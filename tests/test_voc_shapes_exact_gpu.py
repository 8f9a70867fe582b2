"""-m gpu: the benchmark's c4 step (VOC-shaped images through dino_vits16, K = 5, ViT sub-batches of 128) checked as
closely as the default configuration. The step is derived as bench.run_c4 derives it: the first 528 indices of rank 0's
shard of synth.voc_shapes(50_000, seed=0), grouped by shape. That gives eight groups with patch grids of N = 527 to
961 (T = N + 1 tokens, odd N at 527 and 713). The 375 x 500 group holds 260 images: ViT sub-batches of 128, 128 and
4, and more images than the eigensolver has CTAs in one wave.

- GEMMs bit for bit (test_vit_exact_gpu._gemm_case, integer operands) at every distinct T with the largest sub-batch
  of that T, and at the 4-image tail: the PATCH (rin = N) and DROPCLS (rin = T) row remaps at odd rin. The ping-pong
  and cooperative schedules agree at 128 x 714.
- Attention against float64 at T = 528, 621, 661, 714 and 962, 6 heads; every image bitwise the image alone.
- forward_k of every sub-batch of the step: selected images bitwise the image alone; two images per shape against the
  fp32 oracle.
- The step's affinities (zero pad columns, bitwise per image) and eigensolves against a float64 eigh of each image's
  own affinity (test_eigsh_edges_gpu._check); the 260-image group bitwise its solo solves.
- The c4 arrangement, one DinoViT shared by one SpectralPipeline per group, in both group orders over NaN-poisoned
  workspaces; run_host and run_host_pipelined against run_device.
- extract_all over a list of PNGs of all eight shapes: every file against forward_k of its image alone and float64,
  the segmentation PNGs' shapes, and the same tensors at batch_size 1."""
import time
from collections import Counter

import numpy as np
import pytest
import torch

from conftest import load_pkg
from test_eigsh_edges_gpu import _check, _same, _solve, _truth
from test_gemm_schedule_gpu import _run as _schedules_agree
from test_vit_exact_gpu import (EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RESID_F32, EPI_DROPCLS_F32, EPI_PATCH_F32,
                                _att_qkv, _att_ref_and_bound, _att_run, _diff, _gemm_case)

pytestmark = pytest.mark.gpu

MODEL, K, VB, P = "dino_vits16", 5, 128, 16     # run_c4: dino_vits16, K = 5, SpectralPipeline(vit_batch=128)


def _c4_groups():
    """[((H, W), images)] of the benchmark's c4 step in run_c4's (sorted) order."""
    synth, pipeline = load_pkg("synth"), load_pkg("pipeline")
    total = 50_000
    shapes = synth.voc_shapes(total, seed=0)
    mine = pipeline.shard_indices(total, 0, 1)[:528]
    return sorted(Counter(shapes[i] for i in mine).items())


GROUPS = _c4_groups()
SHAPES = [key for key, _ in GROUPS]
COUNT = dict(GROUPS)
BIG = max(SHAPES, key=lambda key: COUNT[key])     # 375 x 500: three ViT sub-batches, a second eigensolver wave


def _n(key):
    return (key[0] // P) * (key[1] // P)


def _sub_batches(B):
    return [(s, min(s + VB, B)) for s in range(0, B, VB)]


def _sid(key):
    return f"{key[0]}x{key[1]}"


@pytest.fixture(scope="module", autouse=True)
def _report(cuda):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    print(f"\ntest_voc_shapes_exact_gpu: {time.perf_counter() - t0:.1f} s, "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def test_c4_step_table(cuda):
    """The step this file checks is the one the benchmark times, and it still has a tail sub-batch and a second wave."""
    assert sum(COUNT.values()) == 528 and len(GROUPS) == 8
    assert [c for c in COUNT.values() if c > VB] == [COUNT[BIG]] and COUNT[BIG] % VB != 0
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    assert COUNT[BIG] > sms, f"the {_sid(BIG)} group ({COUNT[BIG]} images) no longer fills a second wave of {sms} SMs"
    for key, cnt in GROUPS:
        print(f"{_sid(key)}: {cnt} images, N={_n(key)}, T={_n(key) + 1}, pitch={load_pkg('spectral').pitch(_n(key))}, "
              f"sub-batches {[e - s for s, e in _sub_batches(cnt)]}")


# ---------------------------------------------------------------------------------------------------------------
# GEMMs bit for bit
def _step_gemms(tag, B, T):
    N = T - 1
    return [(f"{tag}-qkv", EPI_BIAS_F16, B * T, 1152, 384, 0, 0),
            (f"{tag}-proj", EPI_BIAS_RESID_F32, B * T, 384, 384, 0, 0),
            (f"{tag}-fc1", EPI_BIAS_GELU_F16, B * T, 1536, 384, 0, 0),
            (f"{tag}-fc2", EPI_BIAS_RESID_F32, B * T, 384, 1536, 0, 0),
            (f"{tag}-patch", EPI_PATCH_F32, B * N, 384, 768, N, T),
            (f"{tag}-kproj", EPI_DROPCLS_F32, B * T, 384, 384, T, N)]


def _largest_sub_batch_per_t():
    out = {}
    for key, cnt in GROUPS:
        T = _n(key) + 1
        out[T] = max(out.get(T, 0), min(cnt, VB))
    return sorted(out.items())


TS = [T for T, _ in _largest_sub_batch_per_t()]
STEP_GEMMS = [c for T, B in _largest_sub_batch_per_t() for c in _step_gemms(f"T{T}x{B}", B, T)] + \
    _step_gemms(f"tail-T{_n(BIG) + 1}x{COUNT[BIG] % VB}", COUNT[BIG] % VB, _n(BIG) + 1)


@pytest.mark.parametrize("name,epi,M,N,K,rin,rout", STEP_GEMMS, ids=[c[0] for c in STEP_GEMMS])
def test_gemm_exact_c4_step_shapes(cuda, name, epi, M, N, K, rin, rout):
    _gemm_case(cuda, epi, M, N, K, seed=len(name) * 1000 + M + N + K + epi, rin=rin, rout=rout)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name,epi,N,K", [("fc1", EPI_BIAS_GELU_F16, 1536, 384), ("fc2", EPI_BIAS_RESID_F32, 384, 1536)])
def test_schedules_agree_c4(cuda, name, epi, N, K):
    _schedules_agree(cuda, epi, VB * (_n(BIG) + 1), N, K, seed=N + K + epi + 714)
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# attention against float64
@pytest.mark.parametrize("T", TS)
def test_attention_c4_float64_bound_and_batch_independence(cuda, T):
    """5 images x 6 heads at every token count of the step (test_vit_exact_gpu._att_qkv: odd images with x30 keys and
    +-60000 values next to even ones, rows aimed at the first, middle and last key)."""
    B, heads = 5, 6
    qkv = _att_qkv(B, T, heads, seed=T * 31 + heads, dev=cuda)
    out = _att_run(qkv, B, T, heads)
    o, bound = _att_ref_and_bound(qkv, B, T, heads)
    err = (out.double() - o).abs()
    ok = err <= bound          # NaN fails
    worst = float((err / bound).max())
    print(f"attention T={T} heads={heads}: worst err/bound {worst:.3f} (margin {1 - worst:.3f}), "
          f"max err {float(err.max()):.3e}")
    assert ok.all(), f"attention beyond its rounding bound: {_diff(~ok)}; worst err/bound {worst:.2f}"
    for b in range(B):
        alone = _att_run(qkv[b * T:(b + 1) * T].contiguous(), 1, T, heads)
        assert torch.equal(alone, out[b * T:(b + 1) * T]), f"image {b} differs when run alone"


# ---------------------------------------------------------------------------------------------------------------
# the step computed directly: forward_k in sub-batches of 128, affinity with its epilogue degree, one solve per group
@pytest.fixture(scope="module")
def state_dict():
    return load_pkg("vit").random_state_dict(MODEL, 0)      # what extract_all(seed=0) loads


@pytest.fixture(scope="module")
def model(cuda, state_dict):
    return load_pkg("vit").DinoViT(MODEL, state_dict, device=cuda)


def _images(key, n, seed0=None):
    H, W = key
    return load_pkg("synth").blobs_batch(n, H, W, seed0=1000 * H + W if seed0 is None else seed0)


def _forward_k(model, dev_imgs):
    return torch.cat([model.forward_k(dev_imgs[s:e]) for s, e in _sub_batches(dev_imgs.shape[0])])


@pytest.fixture(scope="module")
def step(cuda, model):
    spectral = load_pkg("spectral")
    out = {}
    for key, cnt in GROUPS:
        imgs = _images(key, cnt)
        feats = _forward_k(model, imgs.to(cuda))
        N = _n(key)
        assert tuple(feats.shape) == (cnt, N, 384) and torch.isfinite(feats).all()
        deg = torch.empty(cnt, N, device=cuda)
        Wm = spectral.affinity(feats, degree=deg)
        eigs = _solve(Wm, N, K, 0, degree=deg)
        out[key] = {"imgs": imgs, "feats": feats, "W": Wm, "deg": deg, "eigs": eigs}
    return out


@pytest.fixture(scope="module")
def ref_vit(cuda, state_dict):
    from oracle import dino_vit
    ref = dino_vit.build(MODEL, seed=0)
    ref.load_state_dict(state_dict)
    return ref.to(cuda)


@pytest.mark.parametrize("key", SHAPES, ids=_sid)
def test_forward_k_c4_batch_equals_single_images(cuda, model, ref_vit, step, key):
    """Every sub-batch of the group (the first is the whole group except at 375 x 500): its first, second, middle and
    last image bitwise the image alone; the group's first and last image against the fp32 oracle."""
    from oracle import dino_vit
    imgs, feats = step[key]["imgs"], step[key]["feats"]
    for s, e in _sub_batches(imgs.shape[0]):
        for i in sorted({s, s + 1, (s + e) // 2, e - 1}):
            k1 = model.forward_k(imgs[i:i + 1].to(cuda))
            assert torch.equal(k1[0], feats[i]), f"{_sid(key)}: image {i} of sub-batch [{s}, {e}) differs when run alone"
    pick = [0, imgs.shape[0] - 1]
    k_ref = torch.cat([ref_vit.forward_k(dino_vit.preprocess_u8(imgs[i], P).to(cuda)) for i in pick])
    k = feats[pick]
    rel = ((k - k_ref).norm() / k_ref.norm()).item()
    cos = torch.nn.functional.cosine_similarity(k.flatten(0, 1), k_ref.flatten(0, 1), dim=-1).min().item()
    print(f"K features {_sid(key)}: rel-L2 {rel:.3e}, min row cosine {cos:.6f}")
    assert rel <= 3e-3 and cos >= 0.9999


# ---------------------------------------------------------------------------------------------------------------
# affinity and eigensolves of the whole step against float64
def test_affinity_c4_pad_columns_and_single_images(cuda, step):
    spectral = load_pkg("spectral")
    for key in SHAPES:
        Wm, N = step[key]["W"], _n(key)
        assert Wm.shape[2] == spectral.pitch(N)
        assert not Wm[:, :, N:].any(), f"{_sid(key)}: pad columns [{N}, {Wm.shape[2]}) are not zero"
        assert torch.isfinite(Wm).all()
    g = step[BIG]
    cnt, N = COUNT[BIG], _n(BIG)
    for i in sorted(set(np.linspace(0, cnt - 1, 9).round().astype(int).tolist()) | {VB - 1, VB, 2 * VB}):
        deg = torch.empty(1, N, device=cuda)
        one = spectral.affinity(g["feats"][i:i + 1], degree=deg)
        assert torch.equal(one[0], g["W"][i]), f"{_sid(BIG)}: affinity of image {i} differs when built alone"
        assert torch.equal(deg[0], g["deg"][i]), f"{_sid(BIG)}: degree of image {i} differs when built alone"


@pytest.mark.parametrize("key", SHAPES, ids=_sid)
def test_eigs_c4_vs_float64(cuda, step, key):
    """Every image of the group, solved as one batch, against a float64 eigh of its own fp32 affinity."""
    g, N = step[key], _n(key)
    ev, vec, info, _ = g["eigs"]
    worst = 0.0
    for i in range(COUNT[key]):
        worst = max(worst, _check(ev[i], vec[i], info[i], _truth(g["W"][i:i + 1], N, 0), K, f"{_sid(key)} image {i}"))
    steps = info[:, 0].float()
    print(f"{_sid(key)} ({COUNT[key]} images, N={N}): Lanczos steps {int(steps.min())}-{int(steps.max())}, "
          f"worst _check ratio {worst:.3f}")


def test_eigs_c4_second_wave_matches_single_image_solves(cuda, step):
    g, N = step[BIG], _n(BIG)
    for i in range(COUNT[BIG]):
        one = _solve(g["W"][i:i + 1], N, K, 0, degree=g["deg"][i:i + 1])
        _same(tuple(t[i:i + 1] for t in g["eigs"]), one, f"{_sid(BIG)} image {i} of {COUNT[BIG]}")


# ---------------------------------------------------------------------------------------------------------------
# the c4 arrangement and the host-buffer drivers
def _outputs(out):
    return tuple(t.clone() for t in out)


def test_c4_arrangement_both_orders(cuda, state_dict, step, monkeypatch):
    """One DinoViT shared by one SpectralPipeline per group, as run_c4 builds them, starting from empty workspaces (a
    new model and a new spectral scratch), so they grow in sorted order. Then the shared ViT workspace, the spectral
    scratch and every pipeline's affinity buffer are filled with NaN bytes, the ViT workspace is cut back to what the
    first group of the reverse order needs (it grows again at a later group), and the step runs in reverse order.
    Both runs, a fresh pipeline per group and the direct calls of the `step` fixture must agree bit for bit; so must
    run_host from pinned memory."""
    pipeline, spectral, vit = load_pkg("pipeline"), load_pkg("spectral"), load_pkg("vit")
    monkeypatch.setattr(spectral, "_scratch", spectral._Scratch())
    shared = vit.DinoViT(MODEL, state_dict, device=cuda)
    devi = {key: step[key]["imgs"].to(cuda) for key in SHAPES}
    pipes = {key: pipeline.SpectralPipeline(MODEL, K=K, device=cuda, vit_batch=VB, model=shared) for key in SHAPES}

    def run(order):
        return {key: _outputs(pipes[key].run_device(devi[key])) for key in order}

    first = run(SHAPES)
    torch.cuda.synchronize()
    shared._ws.fill_(0xFF)
    last = SHAPES[-1]
    need = int(shared.lib.dss_vit_workspace_bytes(shared._h, min(COUNT[last], VB), last[0], last[1]))
    assert need < shared._ws.numel()
    shared._ws = shared._ws[:need]
    for b in spectral._scratch.bufs.values():
        b.fill_(0xFF)
    for p in pipes.values():
        p._bufs["W"].view(torch.uint8).fill_(0xFF)
    second = run(SHAPES[::-1])
    assert shared._ws.numel() > need, "the ViT workspace did not grow during the reverse run"
    for key in SHAPES:
        _same(first[key], second[key], f"{_sid(key)}: sorted vs reverse order")
        _same(first[key], step[key]["eigs"][:3], f"{_sid(key)}: pipeline vs direct forward_k / affinity / eigsh")
        alone = pipeline.SpectralPipeline(MODEL, K=K, device=cuda, vit_batch=VB, model=shared)
        _same(first[key], _outputs(alone.run_device(devi[key])), f"{_sid(key)}: shared pipelines vs a fresh one")
        host = pipes[key].run_host(step[key]["imgs"].pin_memory())
        _same(tuple(t.cpu() for t in first[key]), host, f"{_sid(key)}: run_host vs run_device")
        del alone


def test_run_host_pipelined_c4(cuda, model):
    """Three distinct 160-image 375 x 500 batches (two ViT sub-batches each) through the streaming driver: each yield,
    compared when it is yielded, is bitwise run_device of its batch and its features bitwise forward_k."""
    pipeline = load_pkg("pipeline")
    n = 160
    batches = [_images(BIG, n, seed0=500_000 + 1000 * b) for b in range(3)]
    ref_pipe = pipeline.SpectralPipeline(MODEL, K=K, device=cuda, vit_batch=VB, model=model)
    want = []
    for hb in batches:
        d = hb.to(cuda)
        want.append((tuple(t.cpu() for t in ref_pipe.run_device(d)), _forward_k(model, d).cpu()))
    pipe = pipeline.SpectralPipeline(MODEL, K=K, device=cuda, vit_batch=VB, model=model)
    got = 0
    for i, out in enumerate(pipe.run_host_pipelined([b.pin_memory() for b in batches], features=True)):
        assert i < len(batches), "more yields than batches"
        _same(want[i][0], out[:3], f"run_host_pipelined batch {i}")
        assert torch.equal(out[3], want[i][1]), f"run_host_pipelined batch {i}: features differ from forward_k"
        got += 1
    assert got == len(batches)


# ---------------------------------------------------------------------------------------------------------------
# extract_all over a mixed-shape list
def test_extract_all_c4_mixed_shapes(cuda, model, tmp_path, monkeypatch):
    """PNGs (lossless: the decoded pixels are the synth image) of all eight shapes, interleaved in the sorted list: 3 of
    each, and 3 more of 375 x 500 and 500 x 375 so that those two fill a batch of 4. One decode thread keeps the
    batching deterministic, and the assembler closes its largest open batch beyond 12 pending images (8 x batch_size
    by default, which 8 shapes of at most 3 open rows each never reach), so the run sees full batches, batches closed
    early and partial batches at the end. Every written file is checked against the image alone; a second run at
    batch_size 1 must write the same tensors."""
    from PIL import Image
    from oracle import segment_ref
    extract, io_pipeline, spectral, synth = (load_pkg(m) for m in ("extract", "io_pipeline", "spectral", "synth"))
    root = tmp_path / "images"
    root.mkdir()
    order = [key for _ in range(3) for key in SHAPES] + [BIG, (BIG[1], BIG[0])] * 3
    assert (BIG[1], BIG[0]) in SHAPES
    imgs = {}
    for j, key in enumerate(order):
        stem = f"im{j:03d}"
        imgs[stem] = synth.blobs_image(key[0], key[1], 900_000 + j)
        Image.fromarray(imgs[stem].numpy()).save(root / f"{stem}.png")
    (tmp_path / "list.txt").write_text("".join(f"{s}.png\n" for s in imgs))
    batches = []

    class Assembler(io_pipeline.BatchAssembler):
        def __init__(self, *args, **kwargs):
            super().__init__(*args, **{**kwargs, "max_pending": 12})

        def __iter__(self):
            for b in super().__iter__():
                batches.append((b.key, len(b.items)))
                yield b

    monkeypatch.setattr(io_pipeline, "BatchAssembler", Assembler)
    runs = {}
    for bs in (4, 1):
        d = {n: tmp_path / f"{n}{bs}" for n in ("features", "eigs", "single", "multi")}
        batches.clear()
        extract.extract_all(str(tmp_path / "list.txt"), str(root), MODEL, str(d["features"]), str(d["eigs"]), K=K,
                            batch_size=bs, seed=0, single_region_dir=str(d["single"]), multi_region_dir=str(d["multi"]),
                            num_workers=1)
        assert sum(c for _, c in batches) == len(order) and max(c for _, c in batches) == bs
        runs[bs] = d
        if bs == 4:
            print(f"extract_all batch_size=4 batches: {[(_sid(k_), c) for k_, c in batches]}")
            first_batch = {}
            for k_, c in batches:
                first_batch.setdefault(k_, c)
            assert any(c == 4 for _, c in batches), "no full batch"
            assert any(c < 4 and Counter(k_ for k_, _ in batches)[k_] > 1 for k_, c in first_batch.items()), \
                "no batch closed before its shape's images ran out"
    d = runs[4]
    for dname in d.values():
        assert sorted(p.stem for p in dname.iterdir()) == sorted(imgs), dname
    worst = {}
    info = torch.tensor([0, 1, 0, 0], dtype=torch.int32)
    for j, (stem, img) in enumerate(imgs.items()):
        H, W = order[j]
        Hp, Wp = H // P, W // P
        N = Hp * Wp
        f = torch.load(d["features"] / f"{stem}.pth")
        assert f["shape"] == (1, 3, H, W) and f["file"] == f"{stem}.png" and f["id"] == stem, (stem, f["shape"])
        assert tuple(f["k"].shape) == (1, N, 384) and f["k"].dtype == torch.float32
        k1 = model.forward_k(img[None].to(cuda))
        assert torch.equal(f["k"][0], k1[0].cpu()), f"{stem} ({H}x{W}): features differ from the image alone"
        e = torch.load(d["eigs"] / f"{stem}.pth")
        ev, vec = e["eigenvalues"], e["eigenvectors"]
        assert tuple(ev.shape) == (K,) and tuple(vec.shape) == (K, N)
        deg = torch.empty(1, N, device=cuda)
        Wm = spectral.affinity(f["k"].to(cuda), degree=deg)
        r = _check(ev, vec, info, _truth(Wm, N, 0), K, f"extract_all {stem} ({H}x{W})")
        worst[(H, W)] = max(worst.get((H, W), 0.0), r)
        single = np.array(Image.open(d["single"] / f"{stem}.png"))
        assert single.shape == (Hp, Wp), (stem, single.shape)
        assert np.array_equal(single, segment_ref.single_region(vec.numpy(), Hp, Wp, 0.0)), stem
        multi = np.array(Image.open(d["multi"] / f"{stem}.png"))
        assert multi.shape == (Hp, Wp), (stem, multi.shape)
        f1 = torch.load(runs[1]["features"] / f"{stem}.pth")
        e1 = torch.load(runs[1]["eigs"] / f"{stem}.pth")
        assert torch.equal(f1["k"], f["k"]), f"{stem}: features differ between batch_size 4 and 1"
        assert torch.equal(e1["eigenvalues"], ev) and torch.equal(e1["eigenvectors"], vec), \
            f"{stem}: eigs differ between batch_size 4 and 1"
    print("extract_all worst _check ratio per shape: " + ", ".join(f"{_sid(k_)} {v:.3f}" for k_, v in sorted(worst.items())))
