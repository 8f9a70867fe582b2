"""-m gpu: the eigensolver's paired instantiations against float64, through dss_debug_eigsh.

csrc/eigsh.cu compiles lanczos_laplacian_kernel three times: <4, 1, 512> (variant 2, the default), <2, 2, 512> (variant 1)
and <4, 2, 256> (variant 3). The paired ones run two CTAs per SM with their own rows per warp and pass, load-group
width, warp count (so their own order of combining the column accumulators and every block sum) and grid (2 x SMs
CTAs, each with its own basis slice). Here they get the edge battery of test_eigsh_edges_gpu.py, with its float64 truth
and tolerances, and the geometry of the pairing itself: batches around 2 x SMs, the benchmark's step, the shared-memory
limit of the pairing and the workspace it needs. Variant 2 through the debug entry is the control: bitwise the product
entry points."""
import numpy as np
import pytest
import torch

from conftest import load_pkg
from test_eigsh_edges_gpu import (A_SIZES, CLIQUE_SIZE, _check, _cliques, _covariance, _degree, _dense_random, _dev,
                                  _lattice, _same, _sbm, _simple, _solve, _structured, _truth)

pytestmark = pytest.mark.gpu

VARIANTS = [1, 3]                       # <2, 2, 512>, <4, 2, 256>
VNAME = {1: "<2,2,512>", 2: "<4,1,512>", 3: "<4,2,256>"}
ERR_WORKSPACE, ERR_UNSUPPORTED = -3, -4
WORST = {}                              # variant -> worst _check ratio (error / tolerance) seen in this module


def _lib():
    _l = load_pkg("_lib")
    return _l, _l.load()


def _vsolve(Wm, N, K, mode, variant, degree=None, max_steps=0):
    """dss_debug_eigsh with the instantiation forced: (evals, evecs, info, resid) as spectral.eigsh_* returns them."""
    _l, lib = _lib()
    B, _, ldw = Wm.shape
    dev = Wm.device
    evals = torch.full((B, K), float("nan"), device=dev)
    evecs = torch.full((B, K, N), float("nan"), device=dev)
    info = torch.full((B, 4), -1, dtype=torch.int32, device=dev)
    resid = torch.full((B, K), float("nan"), device=dev)
    need = int(lib.dss_debug_eigsh_workspace_bytes(B, N, K, max_steps, variant))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    _l.check(lib.dss_debug_eigsh(Wm.data_ptr(), _l.ptr(degree), ldw, B, N, K, mode, 0.0, max_steps, variant,
                                 evals.data_ptr(), evecs.data_ptr(), info.data_ptr(), resid.data_ptr(), ws.data_ptr(),
                                 need, _l.stream_ptr()), f"dss_debug_eigsh variant {variant}")
    torch.cuda.synchronize()
    return evals, evecs, info, resid


def _vsolve_retry(Wm, N, K, mode, variant, degree=None):
    """test_eigsh_edges_gpu._solve_retry under the forced variant: the default budget, then the largest Krylov space."""
    out = _vsolve(Wm, N, K, mode, variant, degree)
    if int(out[2][0, 1]) != 1:
        out = _vsolve(Wm, N, K, mode, variant, degree, max_steps=N - 1)
    return out


def _vcheck(variant, ev, vec, info, truth, K, what):
    worst = _check(ev, vec, info, truth, K, f"variant {variant} {what}")
    WORST[variant] = max(WORST.get(variant, 0.0), worst)
    return worst


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    for v in sorted(WORST):
        print(f"variant {v} {VNAME[v]}: worst _check error / tolerance {WORST[v]:.3f}")


# ---------------------------------------------------------------------------------------------------------------
# control: variant 2 through the debug entry is the product path

@pytest.mark.parametrize("case", ["structured196", "structured1025", "sbm515", "cliques4"])
def test_variant2_is_bitwise_the_product_path(cuda, case):
    if case.startswith("structured"):
        N = int(case[len("structured"):])
        Wm, deg = _structured(N, seed=N + 5)
    else:
        Wm = _dev(_sbm(515, seed=3) if case == "sbm515" else _cliques(4, 40, 1e-3))
        N = Wm.shape[1]
        deg = _degree(Wm, N)
    for mode in (0, 1, 2):
        for dg in ((deg, None) if mode != 2 else (None,)):
            ref = _solve(Wm, N, 5, mode, degree=dg)
            got = _vsolve(Wm, N, 5, mode, 2, degree=dg)
            _same(ref, got, f"{case} mode={mode} degree={'given' if dg is not None else 'computed'}")


# ---------------------------------------------------------------------------------------------------------------
# A. strip and padding geometry

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["structured", "sbm"])
@pytest.mark.parametrize("N", A_SIZES)
def test_geometry_vs_float64(cuda, N, kind, variant):
    if kind == "sbm" and N % 4 == 0:
        pytest.skip("the random graph covers the padded widths")
    K = min(5, N - 1)
    if kind == "structured":
        Wm, deg = _structured(N, seed=N)
    else:
        Wm = _dev(_sbm(N, seed=N))
        deg = _degree(Wm, N)
    for mode in (0, 1):
        truth = _truth(Wm, N, mode)
        for dg in (deg, None):
            ev, vec, info, _ = _vsolve(Wm, N, K, mode, variant, degree=dg)
            what = f"{kind} N={N} mode={mode} degree={'given' if dg is not None else 'computed'}"
            _vcheck(variant, ev[0], vec[0], info[0], truth, K, what)
            if kind == "structured" and _simple(truth, K):
                assert int(info[0, 3]) == 0, f"{what}: restarted on an ordinary spectrum, info {info[0].tolist()}"


# ---------------------------------------------------------------------------------------------------------------
# B. what the kernel must not read

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N", [513, 1023])
def test_lower_triangle_and_row_tail_are_not_read(cuda, N, mode, variant):
    spectral = load_pkg("spectral")
    K = 5
    Wm, deg = _structured(N, seed=7 + N)
    dg = deg if mode != 2 else None
    ref = _vsolve(Wm, N, K, mode, variant, degree=dg)
    assert int(ref[2][0, 1]) == 1
    low = Wm.clone()
    r, c = torch.tril_indices(N, N, -1, device=Wm.device)
    low[0, r, c] = float("nan")
    _same(ref, _vsolve(low, N, K, mode, variant, degree=dg), f"variant {variant} N={N} mode={mode} lower triangle NaN")
    P = spectral.pitch(N)
    wide = torch.full((1, N, P + 8), float("nan"), device=Wm.device)
    wide[:, :, :P] = Wm
    _same(ref, _vsolve(wide, N, K, mode, variant, degree=dg), f"variant {variant} N={N} mode={mode} row tail NaN")
    if mode != 2:
        _same(_vsolve(Wm, N, K, mode, variant), _vsolve(wide, N, K, mode, variant),
              f"variant {variant} N={N} mode={mode} degree computed, row tail NaN")


# ---------------------------------------------------------------------------------------------------------------
# C. K edges

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1])
def test_k1_is_the_analytic_null_pair(cuda, mode, variant):
    N = 196
    Wm, deg = _structured(N, seed=3)
    ev, vec, info, _ = _vsolve(Wm, N, 1, mode, variant, degree=deg)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, mode), 1, f"K=1 mode={mode}")
    assert float(ev[0, 0]) == 0.0 and int(info[0, 0]) == 0
    c0 = 1.0 / float(deg.double().sum()) ** 0.5 if mode == 0 else 1.0 / N ** 0.5
    assert (vec[0, 0].double() - c0).abs().max().item() <= 1e-6 * c0


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_k2(cuda, mode, variant):
    N = 196
    Wm, deg = _structured(N, seed=4)
    ev, vec, info, _ = _vsolve(Wm, N, 2, mode, variant, degree=deg if mode != 2 else None)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, mode), 2, f"K=2 mode={mode}")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1])
def test_k64_at_n900(cuda, mode, variant):
    N = 900
    Wm = _dev(_lattice(30, 30, jitter=0.2, seed=1))
    ev, vec, info, _ = _vsolve(Wm, N, 64, mode, variant, degree=_degree(Wm, N), max_steps=N - 1)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, mode), 64, f"K=64 N=900 mode={mode}")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N", [6, 9, 17])
def test_k_is_n_minus_1_whole_spectrum(cuda, N, mode, variant):
    Wm = _dev(_dense_random(N, seed=N, signed=mode == 2))
    ev, vec, info, _ = _vsolve(Wm, N, N - 1, mode, variant, degree=_degree(Wm, N) if mode != 2 else None)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, mode), N - 1, f"K=N-1 N={N} mode={mode}")


@pytest.mark.parametrize("variant", VARIANTS)
def test_topk_k64_at_d100(cuda, variant):
    d = 100
    Wm = _dev(_covariance(d, np.geomspace(10.0, 0.01, d), seed=5))
    ev, vec, info, _ = _vsolve(Wm, d, 64, 2, variant)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, d, 2), 64, "topk K=64 d=100")


# ---------------------------------------------------------------------------------------------------------------
# D. degenerate spectra and breakdown

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("K", [5, 8])
@pytest.mark.parametrize("eps", [0.0, 1e-3])
@pytest.mark.parametrize("c", [3, 4, 6, 8])
def test_cliques_exact_multiplicities(cuda, c, eps, K, mode, variant):
    Wm = _dev(_cliques(c, CLIQUE_SIZE[c], eps))
    N = Wm.shape[1]
    ev, vec, info, _ = _vsolve_retry(Wm, N, K, mode, variant, degree=_degree(Wm, N) if mode != 2 else None)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, mode), K, f"{c} cliques eps={eps} K={K} mode={mode}")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("K", [5, 8])
@pytest.mark.parametrize("hw", [(30, 30), (23, 31)])
def test_lattice(cuda, hw, K, mode, variant, request):
    """The square grid's double eigenvalues: the default instantiation misses a copy at K = 5 in the Laplacian modes
    (a strict xfail in test_eigsh_edges_gpu.py). Whether another instantiation does depends on its rounding, so that
    case is run without pinning the outcome either way, and the outcome is printed."""
    unpinned = hw == (30, 30) and K == 5 and mode in (0, 1)
    if unpinned:
        request.applymarker(pytest.mark.xfail(strict=False, reason="a copy of a double eigenvalue may be missed"))
    Wm = _dev(_lattice(*hw))
    N = Wm.shape[1]
    ev, vec, info, _ = _vsolve_retry(Wm, N, K, mode, variant, degree=_degree(Wm, N) if mode != 2 else None)
    try:
        _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, mode), K, f"lattice {hw} K={K} mode={mode}")
    except AssertionError as e:
        if unpinned:
            print(f"variant {variant} lattice {hw} K={K} mode={mode}: misses a copy ({e})")
        raise
    if unpinned:
        print(f"variant {variant} lattice {hw} K={K} mode={mode}: finds both copies, info {info[0].tolist()}")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("spectrum", ["rank3", "rank10", "isotropic_plus_rank3"])
def test_topk_rank_deficient_covariance(cuda, spectrum, variant):
    d, K = 100, 16
    top = np.linspace(5.0, 1.5, 10)
    s = {"rank3": np.r_[top[:3], np.zeros(d - 3)], "rank10": np.r_[top, np.zeros(d - 10)],
         "isotropic_plus_rank3": np.r_[top[:3] + 0.5, np.full(d - 3, 0.5)]}[spectrum]
    Wm = _dev(_covariance(d, s, seed=11))
    ev, vec, info, _ = _vsolve_retry(Wm, d, K, 2, variant)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, d, 2), K, f"topk {spectrum}")


# ---------------------------------------------------------------------------------------------------------------
# E. budget exhausted

@pytest.mark.parametrize("variant", VARIANTS)
def test_budget_exhausted_then_retry_converges(cuda, variant):
    extract = load_pkg("extract")
    N, K = 900, 5
    Wm = _dev(_lattice(30, 30, jitter=0.01, seed=2))
    deg = _degree(Wm, N)
    ev, vec, info, _ = _vsolve(Wm, N, K, 0, variant, degree=deg, max_steps=12)
    assert int(info[0, 1]) == 0 and int(info[0, 0]) == 12, info[0].tolist()

    def solve(sel, max_steps):
        return _vsolve(Wm, N, K, 0, variant, degree=deg, max_steps=max_steps or 12)[:3]

    ev, vec, info, failed = extract._solve_with_retry(solve, 1, N)
    assert failed == []
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, 0), K, "retry after an exhausted budget")


# ---------------------------------------------------------------------------------------------------------------
# F. the pairing's own geometry: 2 x SMs CTAs, each with its own basis slice

def _batch_vs_solo(Wm, deg, N, K, variant, what):
    B = Wm.shape[0]
    ev, vec, info, res = _vsolve(Wm, N, K, 0, variant, degree=deg)
    assert int(info[:, 1].sum()) == B, f"{what}: {B - int(info[:, 1].sum())} images did not converge"
    for i in range(B):
        one = _vsolve(Wm[i:i + 1], N, K, 0, variant, degree=deg[i:i + 1])
        _same((ev[i:i + 1], vec[i:i + 1], info[i:i + 1], res[i:i + 1]), one, f"{what}: image {i} of {B}")
    for i in np.linspace(0, B - 1, 8).round().astype(int):
        _vcheck(variant, ev[i], vec[i], info[i], _truth(Wm[i:i + 1], N, 0), K, f"{what}: image {i} of {B}")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("extra", [-1, 0, 1, None])
@pytest.mark.parametrize("N", [196, 713])
def test_pairing_waves_match_single_image_solves(cuda, N, extra, variant):
    """B = 2 SMs - 1, 2 SMs, 2 SMs + 1 and 4 SMs + 3: one CTA idle, every CTA busy once, one CTA with a second image,
    every CTA with two or three."""
    spectral, synth = load_pkg("spectral"), load_pkg("synth")
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    B = 2 * sms + extra if extra is not None else 4 * sms + 3
    feats = torch.stack([synth.structured_features(N, 64, 6, 2000 + i) for i in range(B)]).cuda()
    deg = torch.empty(B, N, device=cuda)
    Wm = spectral.affinity(feats, degree=deg)
    _batch_vs_solo(Wm, deg, N, 5, variant, f"variant {variant} N={N} B={B}")


BENCH_B = 264   # images per benchmark step (2 x 132 SMs)


@pytest.mark.parametrize("variant", VARIANTS)
def test_benchmark_step(cuda, variant):
    """The benchmark's eigensolve: 264 images of N = 900 patches with d = 384 structured features, K = 5."""
    spectral, synth = load_pkg("spectral"), load_pkg("synth")
    N = 900
    feats = torch.stack([synth.structured_features(N, 384, 6, 5000 + i) for i in range(BENCH_B)]).cuda()
    deg = torch.empty(BENCH_B, N, device=cuda)
    Wm = spectral.affinity(feats, degree=deg)
    _batch_vs_solo(Wm, deg, N, 5, variant, f"variant {variant} benchmark step")


# ---------------------------------------------------------------------------------------------------------------
# G. the limits of the pairing: shared memory and workspace

def _rc(N, variant, ws_bytes, B=1, K=5, mode=0, buf=None):
    """Return code of the debug entry on an N x N problem whose buffers are all `buf` (nothing may be launched)."""
    _l, lib = _lib()
    p = buf.data_ptr()
    return lib.dss_debug_eigsh(p, None, (N + 3) // 4 * 4, B, N, K, mode, 0.0, 0, variant, p, p, p, None, p, ws_bytes,
                               _l.stream_ptr())


@pytest.mark.parametrize("variant", VARIANTS)
def test_shared_memory_limit_of_the_pairing(cuda, variant):
    """The largest N whose two CTAs share an SM (found by probing: with no workspace a pairing that fits is refused for
    the workspace, one that does not for itself) solves to float64 accuracy; the next N is refused with
    DSS_ERR_UNSUPPORTED and launches nothing."""
    _l, lib = _lib()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=cuda)
    n0 = lib.dss_kernel_launch_count()
    lo, hi = 1024, 8192
    assert _rc(lo, variant, 0, buf=buf) == ERR_WORKSPACE
    assert _rc(hi, variant, 0, buf=buf) == ERR_UNSUPPORTED
    while hi - lo > 1:
        mid = (lo + hi) // 2
        rc = _rc(mid, variant, 0, buf=buf)
        assert rc in (ERR_WORKSPACE, ERR_UNSUPPORTED), rc
        lo, hi = (mid, hi) if rc == ERR_WORKSPACE else (lo, mid)
    assert lib.dss_kernel_launch_count() == n0
    print(f"variant {variant}: N = {lo} is the largest that pairs at the default step budget")
    for mode in (0, 2):    # the Laplacian modes and top-K resolve different step budgets below N = 321 only
        assert _rc(lo, variant, 0, mode=mode, buf=buf) == ERR_WORKSPACE
        assert _rc(hi, variant, 0, mode=mode, buf=buf) == ERR_UNSUPPORTED
    N = lo
    Wm, deg = _structured(N, seed=N)
    ev, vec, info, _ = _vsolve_retry(Wm, N, 5, 0, variant, degree=deg)
    _vcheck(variant, ev[0], vec[0], info[0], _truth(Wm, N, 0), 5, f"N={N}, the last that pairs")
    # the next N with a workspace that would be large enough: refused, nothing launched
    N = hi
    Wm = torch.zeros(1, N, (N + 3) // 4 * 4, device=cuda)
    out = torch.zeros(5 * N + 64, device=cuda)
    need = int(lib.dss_debug_eigsh_workspace_bytes(1, N, 5, 0, variant))
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    n0 = lib.dss_kernel_launch_count()
    rc = lib.dss_debug_eigsh(Wm.data_ptr(), None, Wm.shape[2], 1, N, 5, 0, 0.0, 0, variant, out.data_ptr(),
                             out.data_ptr(), out.data_ptr(), None, ws.data_ptr(), need, _l.stream_ptr())
    assert rc == ERR_UNSUPPORTED and f"N={N}".encode() in lib.dss_last_error(), (rc, lib.dss_last_error())
    assert lib.dss_kernel_launch_count() == n0
    assert int(lib.dss_debug_eigsh_workspace_bytes(1, N, 5, 0, 2)) == int(lib.dss_eigsh_workspace_bytes(1, N, 5, 0))


@pytest.mark.parametrize("variant", VARIANTS)
def test_workspace_of_the_pairing(cuda, variant):
    """The paired grid has up to 2 x SMs CTAs, each with its own basis slice: the debug query covers it (at least the
    product's size, twice the product's basis beyond one wave of SMs), and one byte less is refused before any launch."""
    _l, lib = _lib()
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=cuda)
    n0 = lib.dss_kernel_launch_count()
    for B, N in ((1, 196), (sms, 900), (2 * sms, 900), (4 * sms + 3, 713), (BENCH_B, 900)):
        need = int(lib.dss_debug_eigsh_workspace_bytes(B, N, 5, 0, variant))
        prod = int(lib.dss_eigsh_workspace_bytes(B, N, 5, 0))
        assert need >= prod > 0, (B, N, need, prod)
        if B >= 2 * sms:
            assert need >= 2 * prod - 1024, (B, N, need, prod)
        assert _rc(N, variant, need - 1, B=B, buf=buf) == ERR_WORKSPACE, (B, N)
        assert b"workspace too small" in lib.dss_last_error()
    assert lib.dss_kernel_launch_count() == n0
