"""CPU suite: the C-ABI library loads here (no GPU), exports every symbol include/dss_b200.h declares, validates its
arguments before touching the device, and its host-side positional-embedding interpolation matches upstream DINO."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from conftest import ROOT, load_pkg


def _declared_symbols():
    text = (ROOT / "include" / "dss_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dss_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    _lib = load_pkg("_lib")
    lib = _lib.load()
    names = _declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"libdss_b200.so does not export {n}"
    # and the ctypes prototype table covers the whole header
    assert set(names) == set(_lib.PROTOTYPES), set(names) ^ set(_lib.PROTOTYPES)
    assert lib.dss_version() >= 1


def test_bad_arguments_are_rejected_before_any_device_work():
    _lib = load_pkg("_lib")
    lib = _lib.load()
    n0 = lib.dss_kernel_launch_count()                  # (GPU tests earlier in the same process count too)
    assert lib.dss_affinity(None, 1, 10, 8, 3, None, 0.0, None, 12, None, None, 0, None) == -1
    assert b"null" in lib.dss_last_error()
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    assert lib.dss_affinity(p, 1, 10, 8, 3, None, 0.0, p, 11, None, p, 1 << 15, None) == -1     # ldw not multiple of 4
    assert lib.dss_affinity(p, 1, 10, 8, 3, None, 0.0, p, 12, None, p, 16, None) == -3         # workspace too small
    assert lib.dss_eigsh_laplacian(p, None, 12, 1, 10, 10, 1, 0.0, 0, p, p, p, None, p, 1 << 15, None) == -1   # K >= N
    assert lib.dss_eigsh_laplacian(p, None, 12, 1, 10, 0, 1, 0.0, 0, p, p, p, None, p, 1 << 15, None) == -1    # K < 1
    for variant, mode in ((0, 0), (4, 0), (-1, 2), (3, 3), (1, -1)):                     # forced instantiation
        assert lib.dss_debug_eigsh(p, None, 12, 1, 10, 5, mode, 0.0, 0, variant, p, p, p, None, p, 1 << 15, None) == -1
    assert lib.dss_debug_eigsh_workspace_bytes(1, 10, 5, 0, 0) == 0
    assert lib.dss_debug_eigsh_workspace_bytes(1, 10, 5, 0, 4) == 0
    assert lib.dss_debug_eigsh(p, None, 12, 1, 10, 10, 0, 0.0, 0, 3, p, p, p, None, p, 1 << 15, None) == -1  # K >= N
    for variant in (1, 2, 3):
        need = lib.dss_debug_eigsh_workspace_bytes(300, 700, 5, 0, variant)
        assert need >= lib.dss_eigsh_workspace_bytes(300, 700, 5, 0) > 0
        assert lib.dss_debug_eigsh(p, None, 700, 300, 700, 5, 0, 0.0, 0, variant, p, p, p, None, p, need - 1,
                                   None) == -3                                              # one byte short
    assert lib.dss_debug_eigsh(p, None, 4000, 1, 4000, 5, 0, 0.0, 0, 3, p, p, p, None, p, 1 << 30, None) == -4
    assert b"N=4000" in lib.dss_last_error()                                                # two CTAs do not fit
    assert lib.dss_op_gemm_f16(p, p, p, p, 16, 30, 64, 0, None, 0, 0, None) == -1           # N % 32
    assert lib.dss_op_layernorm_f16(p, p, p, p, 4, 100, 1e-6, None) == -1                   # unsupported width
    cfg = _lib.VitConfig(16, 384, 12, 5, 4, 14, 1e-6)                                       # 384 / 5 != 64
    h = C.c_void_p()
    assert lib.dss_vit_create(C.byref(cfg), C.byref(h)) == -1
    cfg = _lib.VitConfig(16, 384, 12, 6, 4, 14, 1e-6)
    assert lib.dss_vit_create(C.byref(cfg), C.byref(h)) == 0
    assert lib.dss_vit_workspace_bytes(h, 2, 224, 224) > 2 * 197 * 384 * 4
    assert lib.dss_vit_workspace_bytes(h, 2, 8, 224) == 0                                   # smaller than a patch
    assert lib.dss_vit_forward_k(h, p, 1, 224, 224, -1, p, p, 1 << 15, None) == -1          # weights not loaded
    lib.dss_vit_destroy(h)
    assert lib.dss_affinity_workspace_bytes(2, 900, 384) >= 2 * 900 * 384 * 4
    assert lib.dss_kernel_launch_count() == n0                                              # nothing was launched


# mode 0 (mode 2 caps at N). 1602 steps at N = 6400 take exactly the 227 KB less the kernel's 32 B of static shared
# memory; N = 7892 is the largest the default 320 steps fit.
MAX_STEPS = {3600: 3599, 3816: 3815, 3820: 3813, 6400: 1602, 7892: 322, 7896: 319, 7900: 316, 8300: 0}


@pytest.mark.parametrize("N", [3600, 3816, 3817, 3820, 4801, 6400, 7000, 7892, 7893, 7896, 7900, 8300])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_eigsh_max_steps_is_the_largest_budget_that_fits(N, mode):
    """dss_eigsh_max_steps(N, mode) is a budget the solver accepts and, below its cap (N - 1, or N for the plain mode),
    one step more is DSS_ERR_UNSUPPORTED. The shared-memory check runs before the workspace check, so a workspace one
    byte short tells an accepted budget (-3) from a refused one (-4) without any launch."""
    _lib = load_pkg("_lib")
    lib = _lib.load()
    n0 = lib.dss_kernel_launch_count()
    K = 5
    buf = torch.zeros(1 << 12, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    ldw = (N + 3) // 4 * 4

    def call(steps):
        short = lib.dss_eigsh_workspace_bytes(1, N, K, steps) - 1
        if mode == 2:
            return lib.dss_eigsh_topk(p, ldw, 1, N, K, 0.0, steps, p, p, p, None, p, short, None)
        return lib.dss_eigsh_laplacian(p, None, ldw, 1, N, K, 1 - mode, 0.0, steps, p, p, p, None, p, short, None)

    m = lib.dss_eigsh_max_steps(N, mode)
    cap = N if mode == 2 else N - 1
    if N in MAX_STEPS:
        assert m == min(MAX_STEPS[N] + (mode == 2 and MAX_STEPS[N] == N - 1), cap)
    assert 0 <= m <= cap
    if m > 0:
        assert call(m) == -3, lib.dss_last_error()
    if m < cap:
        assert call(m + 1) == -4 and b"shared memory" in lib.dss_last_error()
    if m == 0:   # not even the default budget fits
        assert call(0) == -4
    assert lib.dss_kernel_launch_count() == n0


def test_eigsh_max_steps_rejects_bad_arguments():
    lib = load_pkg("_lib").load()
    assert [lib.dss_eigsh_max_steps(N, mode) for N, mode in ((1, 0), (0, 2), (100, 3), (100, -1))] == [0] * 4
    assert [lib.dss_eigsh_max_steps(2, mode) for mode in (0, 1, 2)] == [1, 1, 2]


@pytest.mark.parametrize("N,budget", [(900, 899), (3600, 3599), (6400, 1602), (7892, 322), (300, None), (7896, None),
                                      (7900, None)])
def test_solve_with_retry_asks_for_the_largest_budget_that_fits(N, budget):
    """The extract commands' retry of non-converged images: the default budget first, then the largest that fits in
    shared memory (not N - 1 above N = 3816); no retry where that is not above the default, the rows reported failed."""
    extract = load_pkg("extract")
    asked = []

    def solve(sel, max_steps):
        asked.append((sel, max_steps))
        B = 3 if sel is None else len(sel)
        info = torch.zeros(B, 4, dtype=torch.int32)
        info[:, 1] = 1 if max_steps else torch.tensor([1, 0, 1][:B])    # row 1 misses the default budget
        return torch.full((B, 2), float(max_steps)), torch.zeros(B, 2, N), info

    evals, _, info, failed = extract._solve_with_retry(solve, 3, N)
    if budget is None:
        assert asked == [(None, 0)] and failed == [1] and int(info[1, 1]) == 0
    else:
        assert asked == [(None, 0), ([1], budget)] and failed == []
        assert evals[:, 0].tolist() == [0.0, float(budget), 0.0] and info[:, 1].tolist() == [1, 1, 1]


@pytest.mark.parametrize("N,budget", [(3600, 3599), (6400, 1602), (7896, None)])
def test_retry_of_a_solved_batch_asks_for_the_largest_budget_that_fits(N, budget):
    """extract_all solves a batch asynchronously and hands the default-budget results to the same retry
    (extract._retry_bad_rows): it re-solves only the bad rows, with the budget that fits, and fills them in place."""
    extract = load_pkg("extract")
    asked = []

    def solve(sel, max_steps):
        asked.append((sel, max_steps))
        info = torch.zeros(len(sel), 4, dtype=torch.int32)
        info[:, 1] = torch.tensor([1, 0, 1])                     # row 2 of the batch fails the retry as well
        return torch.full((len(sel), 2), float(max_steps)), torch.zeros(len(sel), 2, N), info

    evals, evecs, info = torch.zeros(4, 2), torch.zeros(4, 2, N), torch.ones(4, 4, dtype=torch.int32)
    info[[0, 2], 1] = 0
    evecs[3, 0, 5] = float("nan")                                 # converged but non-finite: retried too
    failed = extract._retry_bad_rows(solve, evals, evecs, info, N)
    if budget is None:
        assert asked == [] and failed == [0, 2, 3]
    else:
        assert asked == [([0, 2, 3], budget)] and failed == [2]
        assert evals[:, 0].tolist() == [budget, 0, 0, budget] and info[:, 1].tolist() == [1, 1, 0, 1]


@pytest.mark.parametrize("name,Hp,Wp", [("dino_vits16", 30, 30), ("dino_vits16", 23, 31), ("dino_vits16", 14, 14),
                                        ("dino_vits16", 7, 40), ("dino_vitb8", 60, 60), ("dino_vitb8", 28, 28)])
def test_pos_embed_interpolation_matches_upstream(name, Hp, Wp):
    from oracle import dino_vit
    vit = load_pkg("vit")
    ref = dino_vit.build(name, seed=3)
    P = ref.cfg.patch
    want = ref.interpolate_pos_encoding(Hp * Wp, Hp * P, Wp * P)[0]
    got = vit.pos_embed_interp_host(ref.pos_embed, ref.cfg.grid0, Hp, Wp)
    assert got.shape == want.shape
    assert (got - want).abs().max().item() <= 2e-6


def test_product_path_fails_loudly_without_cuda(tmp_path):
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    _lib = load_pkg("_lib")
    vit = load_pkg("vit")
    spectral = load_pkg("spectral")
    ex = load_pkg("extract")
    with pytest.raises(_lib.DssError):
        vit.get_model("dino_vits16", device="cpu", seed=0)
    with pytest.raises(_lib.DssError, match="pretrained DINO weights not found"):
        vit.get_model("dino_vits16", device="cpu")          # no checkpoint and no explicit opt-in to random weights
    with pytest.raises(_lib.DssError):
        spectral.affinity(torch.zeros(1, 16, 8))
    with pytest.raises(_lib.DssError):
        spectral.eigsh_laplacian(torch.zeros(1, 16, 16), 16, 3)
    (tmp_path / "list.txt").write_text("a.jpg\n")
    with pytest.raises(_lib.DssError):
        ex.extract_features(str(tmp_path / "list.txt"), str(tmp_path), "dino_vits16", 1, str(tmp_path / "out"), seed=0)
    with pytest.raises(ValueError):
        vit.get_model("resnet50")


def test_no_product_module_imports_the_oracle():
    pkg = ROOT / "deep-spectral-segmentation_b200"
    for f in list(pkg.glob("*.py")) + [ROOT / "extract" / "extract.py"]:
        src = f.read_text()
        assert "oracle" not in src.replace("# oracle", ""), f"{f} references the oracle"
