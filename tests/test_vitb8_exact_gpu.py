"""-m gpu: the ViT-B/8 configurations checked as closely as the default one. c3: 480^2 images, T = 3601 tokens,
N = 3600 patches, K = 15 with the colour-KNN term; c5: 640^2, T = 6401, N = 6400, K = 32.

- GEMMs bit for bit at the ViT-B/8 step shapes (test_vit_exact_gpu._gemm_case, integer operands): fc2's K = 3072 runs
  48 slabs through the ring, fc1 writes 3072 columns and qkv 2304. The largest partial sum, 64 * 4 * 3072 = 786432,
  is still below 2^20, so every fp32 sum is exact in any order and the float64 product is THE answer. The ping-pong
  and cooperative schedules must agree bit for bit at c5's fc1 and fc2.
- Attention against float64 at 29 and 51 key tiles (the last one partial: 17 keys and 1 key), with the bound of
  test_vit_exact_gpu._att_ref_and_bound evaluated per (image, head), and every image bitwise the image alone.
- forward_k of c3's 16-image and c5's 8-image batches: selected images bitwise the image alone.
- The eigensolver against a float64 eigh of the kernel's own fp32 affinity of ViT-B/8 features
  (test_eigsh_edges_gpu._check): c3 with the colour term and the epilogue degree, c5, c3's second wave, the largest N
  the default step budget fits, and the retry of an exhausted budget at N = 6400, which needs a budget below N - 1."""
import time

import numpy as np
import pytest
import torch

from conftest import load_pkg
from test_eigsh_edges_gpu import _check, _same, _solve, _solve_retry, _structured, _truth
from test_gemm_schedule_gpu import _run as _schedules_agree
from test_vit_exact_gpu import (EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RESID_F32, EPI_DROPCLS_F32, EPI_PATCH_F32,
                                _att_qkv, _att_ref_and_bound, _att_run, _diff, _gemm_case)

pytestmark = pytest.mark.gpu

C3 = dict(B=16, H=480, T=3601, N=3600, K=15)   # the benchmark's c3 and c5 steps: images per ViT launch sequence
C5 = dict(B=8, H=640, T=6401, N=6400, K=32)
ERR_WORKSPACE, ERR_UNSUPPORTED = -3, -4


@pytest.fixture(scope="module", autouse=True)
def _report(cuda):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    print(f"\ntest_vitb8_exact_gpu: {time.perf_counter() - t0:.1f} s, "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ---------------------------------------------------------------------------------------------------------------
# GEMMs bit for bit
def _step_gemms(tag, B, T):
    P = T - 1
    return [(f"{tag}-qkv", EPI_BIAS_F16, B * T, 2304, 768, 0, 0),
            (f"{tag}-proj", EPI_BIAS_RESID_F32, B * T, 768, 768, 0, 0),
            (f"{tag}-fc1", EPI_BIAS_GELU_F16, B * T, 3072, 768, 0, 0),
            (f"{tag}-fc2", EPI_BIAS_RESID_F32, B * T, 768, 3072, 0, 0),
            (f"{tag}-patch", EPI_PATCH_F32, B * P, 768, 192, P, T),
            (f"{tag}-kproj", EPI_DROPCLS_F32, B * T, 768, 768, T, P)]


STEP_GEMMS = _step_gemms("c3", C3["B"], C3["T"]) + _step_gemms("c5", C5["B"], C5["T"])


@pytest.mark.parametrize("name,epi,M,N,K,rin,rout", STEP_GEMMS, ids=[c[0] for c in STEP_GEMMS])
def test_gemm_exact_vitb8_step_shapes(cuda, name, epi, M, N, K, rin, rout):
    _gemm_case(cuda, epi, M, N, K, seed=len(name) * 1000 + N + K + epi, rin=rin, rout=rout)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name,epi,N,K", [("fc1", EPI_BIAS_GELU_F16, 3072, 768), ("fc2", EPI_BIAS_RESID_F32, 768, 3072)])
def test_schedules_agree_c5(cuda, name, epi, N, K):
    _schedules_agree(cuda, epi, C5["B"] * C5["T"], N, K, seed=N + K + epi)
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# attention against float64
@pytest.mark.parametrize("T", [C3["T"], C5["T"]])
def test_attention_vitb8_float64_bound_and_batch_independence(cuda, T):
    """3 images x 12 heads; the odd image's x30 keys and +-60000 values follow the even ones, rows 2 and 3 of each
    image aim their maximum at key T - 1 (the last, partial key tile) and T // 2. The all-heads float64 scores would
    take tens of GB at T = 6401, so the bound is evaluated one (image, head) at a time."""
    B, heads = 3, 12
    qkv = _att_qkv(B, T, heads, seed=T * 31 + heads, dev=cuda)
    out = _att_run(qkv, B, T, heads)
    per_head = qkv.view(B, T, 3, heads, 64)
    worst, max_err = 0.0, 0.0
    for b in range(B):
        for h in range(heads):
            o, bound = _att_ref_and_bound(per_head[b, :, :, h].reshape(T, 3 * 64), 1, T, 1)
            err = (out[b * T:(b + 1) * T, h * 64:(h + 1) * 64].double() - o).abs()
            ok = err <= bound          # NaN fails
            worst = max(worst, float((err / bound).max()))
            max_err = max(max_err, float(err.max()))
            assert ok.all(), f"image {b} head {h}: beyond the rounding bound: {_diff(~ok)}; worst err/bound {worst:.2f}"
    print(f"attention T={T} heads={heads}: worst err/bound {worst:.3f} (margin {1 - worst:.3f}), max err {max_err:.3e}")
    for b in range(B):
        alone = _att_run(qkv[b * T:(b + 1) * T].contiguous(), 1, T, heads)
        assert torch.equal(alone, out[b * T:(b + 1) * T]), f"image {b} differs when run alone"


# ---------------------------------------------------------------------------------------------------------------
# forward_k: the c3 and c5 batches, and the features the eigensolves below use
@pytest.fixture(scope="module")
def vitb8(cuda):
    model, _, _, _ = load_pkg("vit").get_model("dino_vitb8", seed=0, device=cuda)
    return model


def _features(model, cfg, seed0, dev):
    imgs = load_pkg("synth").blobs_batch(cfg["B"], cfg["H"], cfg["H"], seed0=seed0)
    k = model.forward_k(imgs.to(dev))
    torch.cuda.synchronize()
    assert tuple(k.shape) == (cfg["B"], cfg["N"], 768) and torch.isfinite(k).all()
    return imgs, k


@pytest.fixture(scope="module")
def c3_feats(cuda, vitb8):
    return _features(vitb8, C3, 7, cuda)


@pytest.fixture(scope="module")
def c5_feats(cuda, vitb8):
    return _features(vitb8, C5, 3, cuda)


@pytest.mark.parametrize("cfg", ["c3", "c5"])
def test_forward_k_vitb8_batch_equals_single_images(cuda, vitb8, c3_feats, c5_feats, cfg):
    imgs, k = c3_feats if cfg == "c3" else c5_feats
    B = imgs.shape[0]
    for i in (0, 1, B // 2, B - 1):
        k1 = vitb8.forward_k(imgs[i:i + 1].to(cuda))
        assert torch.equal(k1[0], k[i]), f"{cfg}: image {i} of the {B}-image batch differs from the image alone"


# ---------------------------------------------------------------------------------------------------------------
# eigensolves against float64
def _c3_affinity(imgs, k):
    """The c3 affinity: colour-KNN counts of the 60 x 60 low-resolution image as extract.py:199-204 derives it
    (PIL bilinear of the whole image), lambda = 10, with the epilogue degree."""
    from PIL import Image
    spectral = load_pkg("spectral")
    B, N = k.shape[:2]
    side = int(round(N ** 0.5))
    lr = np.stack([np.array(Image.fromarray(im.numpy()).resize((side, side), Image.BILINEAR)) / 255.0 for im in imgs])
    rgb = torch.from_numpy(lr.reshape(B, N, 3).astype(np.float32)).to(k.device)
    cc = spectral.knn_color_counts(rgb, side, side)
    deg = torch.empty(B, N, device=k.device)
    Wm = spectral.affinity(k, True, True, cc, 10.0, degree=deg)
    del cc
    return Wm, deg


@pytest.mark.parametrize("K", [C3["K"], 32])
def test_c3_eigs_vs_float64(cuda, c3_feats, K):
    """All 16 images of the c3 batch, at c3's K and at K = 32. These spectra have gaps near 1e-4, where a run can return
    K valid eigenpairs that are not the smallest K; the float64 eigenvalues and eigenspaces would show it."""
    imgs, k = c3_feats
    N = C3["N"]
    Wm, deg = _c3_affinity(imgs, k)
    ev, vec, info, _ = _solve(Wm, N, K, 0, degree=deg)
    worst = 0.0
    for i in range(C3["B"]):
        worst = max(worst, _check(ev[i], vec[i], info[i], _truth(Wm[i:i + 1], N, 0), K, f"c3 image {i} K={K}"))
    print(f"c3 K={K}: {info[:, 0].tolist()} Lanczos steps, worst _check ratio {worst:.3f}")


def test_c5_eigs_vs_float64(cuda, c5_feats):
    """All 8 images of the c5 batch, solved as one batch."""
    _, k = c5_feats
    N, K = C5["N"], C5["K"]
    deg = torch.empty(C5["B"], N, device=cuda)
    Wm = load_pkg("spectral").affinity(k, degree=deg)
    ev, vec, info, _ = _solve(Wm, N, K, 0, degree=deg)
    worst = 0.0
    for i in range(C5["B"]):
        worst = max(worst, _check(ev[i], vec[i], info[i], _truth(Wm[i:i + 1], N, 0), K, f"c5 image {i}"))
    print(f"c5: {info[:, 0].tolist()} Lanczos steps, worst _check ratio {worst:.3f}")


def test_c5_retry_after_exhausted_budget(cuda, c5_feats):
    """A first run of only K steps cannot converge at N = 6400; the extract commands' retry must then ask for the
    largest budget that fits in shared memory (N - 1 = 6399 steps does not) and converge."""
    extract, spectral = load_pkg("extract"), load_pkg("spectral")
    _, k = c5_feats
    N, K = C5["N"], C5["K"]
    deg = torch.empty(1, N, device=cuda)
    Wm = spectral.affinity(k[1:2], degree=deg)
    runs = []

    def solve(sel, max_steps):
        out = _solve(Wm, N, K, 0, degree=deg, max_steps=max_steps or K)[:3]
        runs.append((max_steps, out[2].cpu()))
        return out

    ev, vec, info, failed = extract._solve_with_retry(solve, 1, N)
    assert [r[0] for r in runs] == [0, spectral.max_steps(N)], [r[0] for r in runs]
    first = runs[0][1][0]
    assert int(first[1]) == 0 and int(first[0]) == K, f"the {K}-step run reports {first.tolist()}"
    assert failed == [] and 320 < spectral.max_steps(N) < N - 1
    worst = _check(ev[0], vec[0], info[0], _truth(Wm, N, 0), K, "c5 retry")
    print(f"c5 retry: {spectral.max_steps(N)}-step budget, {int(info[0, 0])} steps taken, worst _check ratio {worst:.3f}")


def test_extract_all_retry_at_c5(cuda, tmp_path, monkeypatch):
    """extract_all's own retry (it solves asynchronously, then retries in its second half): a 640^2 image whose first
    solve is limited to K steps must be re-solved with the largest budget that fits at N = 6400, and its eigs file must
    hold the float64 eigenpairs of its features' affinity."""
    from PIL import Image
    extract, spectral = load_pkg("extract"), load_pkg("spectral")
    N, K = C5["N"], C5["K"]
    root = tmp_path / "images"
    root.mkdir()
    Image.fromarray(load_pkg("synth").blobs_image(C5["H"], C5["H"], 11).numpy()).save(root / "img.png")
    (tmp_path / "list.txt").write_text("img.png\n")
    runs = []
    laplacian_eigs = spectral.laplacian_eigs

    def limited(*args, max_steps=0, **kwargs):
        out = laplacian_eigs(*args, max_steps=max_steps or K, **kwargs)
        runs.append((max_steps, out[2].cpu()))
        return out

    monkeypatch.setattr(spectral, "laplacian_eigs", limited)
    extract.extract_all(str(tmp_path / "list.txt"), str(root), "dino_vitb8", str(tmp_path / "f"), str(tmp_path / "e"),
                        K=K, batch_size=1, seed=0)
    assert [r[0] for r in runs] == [0, spectral.max_steps(N)], [r[0] for r in runs]
    assert int(runs[0][1][0, 1]) == 0 and int(runs[1][1][0, 1]) == 1, [r[1][0].tolist() for r in runs]
    eigs = torch.load(tmp_path / "e" / "img.pth")
    k = torch.load(tmp_path / "f" / "img.pth")["k"].reshape(1, N, -1).to(cuda, torch.float32)
    deg = torch.empty(1, N, device=cuda)
    Wm = spectral.affinity(k, degree=deg)
    worst = _check(eigs["eigenvalues"], eigs["eigenvectors"], runs[1][1][0], _truth(Wm, N, 0), K, "extract_all retry")
    print(f"extract_all c5 retry: worst _check ratio {worst:.3f}")


def test_c3_second_wave_matches_single_image_solves(cuda, vitb8):
    """SMs + 1 images at c3's shape (colour term included): the CTA that takes the last image reuses its shared memory
    and scratch. Every image must be bitwise its solo solve; a spread of 8 must pass the float64 check."""
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    B, N, K = sms + 1, C3["N"], C3["K"]
    imgs = load_pkg("synth").blobs_batch(B, C3["H"], C3["H"], seed0=1000)
    k = torch.cat([vitb8.forward_k(imgs[i:i + C3["B"]].to(cuda)) for i in range(0, B, C3["B"])])
    Wm, deg = _c3_affinity(imgs, k)
    del k
    ev, vec, info, res = _solve(Wm, N, K, 0, degree=deg)
    assert int(info[:, 1].sum()) == B, info[:, 1].tolist()
    for i in range(B):
        one = _solve(Wm[i:i + 1], N, K, 0, degree=deg[i:i + 1])
        _same((ev[i:i + 1], vec[i:i + 1], info[i:i + 1], res[i:i + 1]), one, f"image {i} of {B}")
    worst = 0.0
    for i in np.linspace(0, B - 1, 8).round().astype(int):
        worst = max(worst, _check(ev[i], vec[i], info[i], _truth(Wm[i:i + 1], N, 0), K, f"image {i} of {B}"))
    print(f"c3 second wave ({B} images): worst _check ratio {worst:.3f}")
    del Wm
    torch.cuda.empty_cache()


def test_largest_n_at_the_default_budget(cuda):
    """The largest N whose default 320-step solve fits in shared memory, found by probing (the shared-memory check
    comes before the workspace check: with no workspace a fitting N is refused for the workspace, one that does not fit
    for itself), solves to float64 accuracy; the next N (the next padded width) is refused and launches nothing."""
    _l = load_pkg("_lib")
    lib, spectral = _l.load(), load_pkg("spectral")
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=cuda)
    p = buf.data_ptr()

    def rc(N, ws_bytes=0):
        return lib.dss_eigsh_laplacian(p, None, spectral.pitch(N), 1, N, 5, 1, 0.0, 0, p, p, p, None, p, ws_bytes,
                                       _l.stream_ptr())

    n0 = lib.dss_kernel_launch_count()
    lo, hi = 4096, 16384
    assert rc(lo) == ERR_WORKSPACE and rc(hi) == ERR_UNSUPPORTED
    while hi - lo > 1:
        mid = (lo + hi) // 2
        r = rc(mid)
        assert r in (ERR_WORKSPACE, ERR_UNSUPPORTED), r
        lo, hi = (mid, hi) if r == ERR_WORKSPACE else (lo, mid)
    assert lib.dss_kernel_launch_count() == n0
    print(f"N = {lo} is the largest the default step budget fits")
    assert spectral.max_steps(lo) >= spectral.DEFAULT_MAX_STEPS > spectral.max_steps(hi)
    assert spectral.pitch(hi) > spectral.pitch(lo)
    N = lo
    Wm, deg = _structured(N, seed=N)
    ev, vec, info, _ = _solve_retry(Wm, N, 5, 0, degree=deg)
    worst = _check(ev[0], vec[0], info[0], _truth(Wm, N, 0), 5, f"N={N}, the largest at the default budget")
    print(f"N={N}: {int(info[0, 0])} Lanczos steps, worst _check ratio {worst:.3f}")
    del Wm, deg
    # the next N with a workspace that would be large enough: refused, nothing launched
    N = hi
    Wm = torch.zeros(1, N, spectral.pitch(N), device=cuda)
    out = torch.zeros(5 * N + 64, device=cuda)
    need = int(lib.dss_eigsh_workspace_bytes(1, N, 5, 0))
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    n0 = lib.dss_kernel_launch_count()
    r = lib.dss_eigsh_laplacian(Wm.data_ptr(), None, Wm.shape[2], 1, N, 5, 1, 0.0, 0, out.data_ptr(), out.data_ptr(),
                                out.data_ptr(), None, ws.data_ptr(), need, _l.stream_ptr())
    assert r == ERR_UNSUPPORTED and f"N={N}".encode() in lib.dss_last_error(), (r, lib.dss_last_error())
    assert lib.dss_kernel_launch_count() == n0
