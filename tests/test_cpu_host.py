"""CPU suite: host-side logic that mirrors the reference's CLI / file contract (no compute calls)."""
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_pkg


def test_fire_compatible_parser():
    cli = load_pkg("cli")
    ex = load_pkg("extract")
    args, kw = cli.parse_args(ex.extract_eigs, ["--images_root", "imgs", "--features_dir=feat", "--output_dir", "out",
                                               "--which_matrix", "laplacian", "--K", "5", "--nolapnorm",
                                               "--image_color_lambda", "10.0", "--normalize", "False",
                                               "--image_downsample_factor", "None"])
    assert args == [] and kw == {"images_root": "imgs", "features_dir": "feat", "output_dir": "out",
                                 "which_matrix": "laplacian", "K": 5, "lapnorm": False, "image_color_lambda": 10.0,
                                 "normalize": False, "image_downsample_factor": None}
    args, kw = cli.parse_args(ex.extract_features, ["list.txt", "root", "--model_name", "dino_vits16", "--batch_size=1",
                                                   "--output_dir", "o", "--which_block", "-1"])
    assert args == ["list.txt", "root"] and kw["which_block"] == -1 and kw["batch_size"] == 1
    with pytest.raises(SystemExit):
        cli.parse_args(ex.extract_eigs, ["--no_such_flag", "1"])
    with pytest.raises(SystemExit):
        cli.Fire({"extract_eigs": ex.extract_eigs}, ["bogus_command"])
    assert cli.Fire({"f": lambda a, b=2: (a, b)}, ["f", "3", "--b", "[1,2]"]) == (3, [1, 2])


def test_signatures_match_reference_contract():
    """Argument names / defaults of the reference's callables (extract/extract.py:21-28,119-132,247-261)."""
    import inspect
    ex = load_pkg("extract")
    p = inspect.signature(ex.extract_features).parameters
    assert list(p)[:6] == ["images_list", "images_root", "model_name", "batch_size", "output_dir", "which_block"]
    assert p["which_block"].default == -1
    p = inspect.signature(ex.extract_eigs).parameters
    want = {"which_matrix": "laplacian", "which_color_matrix": "knn", "which_features": "k", "normalize": True,
            "threshold_at_zero": True, "lapnorm": True, "K": 20, "image_downsample_factor": None,
            "image_color_lambda": 0.0, "multiprocessing": 0}
    assert list(p)[:3] == ["images_root", "features_dir", "output_dir"]
    for k, v in want.items():
        assert p[k].default == v, k
    p = inspect.signature(ex._extract_eig).parameters
    assert list(p)[:4] == ["inp", "K", "images_root", "output_dir"] and p["image_color_lambda"].default == 10


def test_images_dataset_and_sizes(tmp_path):
    utils = load_pkg("extract_utils")
    synth = load_pkg("synth")
    from PIL import Image
    for name, seed in (("b.png", 1), ("a.png", 2)):
        Image.fromarray(synth.blobs_image(50, 70, seed).numpy()).save(tmp_path / name)
    ds = utils.ImagesDataset(["b.png", "a.png", "b.png"], images_root=str(tmp_path))
    assert ds.filenames == ["a.png", "b.png"] and len(ds) == 2          # de-duplicated + sorted (extract_utils.py:23)
    img, path, idx = ds[0]
    assert path == "a.png" and idx == 0 and img.dtype == torch.uint8 and tuple(img.shape) == (50, 70, 3)
    assert torch.equal(img, synth.blobs_image(50, 70, 2))               # RGB order, lossless png
    d = {"patch_size": 16, "shape": (1, 3, 250, 333)}
    assert utils.get_image_sizes(d) == (1, 3, 250, 333, 16, 15, 20, 240, 320)
    assert utils.get_image_sizes(d, 8)[4:] == (8, 31, 41, 248, 328)


def test_make_output_dir_non_interactive(tmp_path, monkeypatch):
    utils = load_pkg("extract_utils")
    out = tmp_path / "a" / "b"
    utils.make_output_dir(out)
    assert out.is_dir()
    (out / "x.pth").write_text("x")
    utils.make_output_dir(out, assume_yes=True)           # explicit yes
    monkeypatch.setattr(sys.stdin, "isatty", lambda: False, raising=False)
    utils.make_output_dir(out)                             # non-tty: continues instead of blocking on input()
    monkeypatch.setattr(sys.stdin, "isatty", lambda: True, raising=False)
    monkeypatch.setattr("builtins.input", lambda *_: "n")
    with pytest.raises(SystemExit):
        utils.make_output_dir(out)                         # interactive "n" exits like the reference


def test_feature_dict_layout_roundtrips_through_torch_load(tmp_path):
    ex = load_pkg("extract")
    utils = load_pkg("extract_utils")
    k = torch.randn(1, 20 * 15, 384)
    d = ex._feature_dict(k, 7, "sub/img_0007.jpg", "dino_vits16", 16, 250, 333)
    torch.save(d, tmp_path / "f.pth")
    back = torch.load(tmp_path / "f.pth", map_location="cpu")   # weights_only default: the layout must stay loadable
    assert set(back) == {"k", "indices", "file", "id", "model_name", "patch_size", "shape"}
    assert back["id"] == "img_0007" and back["file"][:-4] == "sub/img_0007" and back["indices"].item() == 7
    assert back["indices"].dim() == 0 and back["shape"] == (1, 3, 250, 333) and back["k"].shape == (1, 300, 384)
    assert utils.get_image_sizes(back)[5:7] == (15, 20)


def test_random_state_dict_is_loadable_by_the_oracle_and_deterministic():
    from oracle import dino_vit
    vit = load_pkg("vit")
    sd = vit.random_state_dict("dino_vits16", 0)
    sd2 = vit.random_state_dict("dino_vits16", 0)
    assert all(torch.equal(sd[k], sd2[k]) for k in sd)
    m = dino_vit.DinoViT(dino_vit.cfg_for("dino_vits16"))
    m.load_state_dict(sd)                                   # same parameter names and shapes as upstream
    assert set(vit.flat_param_order("dino_vits16")) == set(sd)   # incl. the final norm (used by forward_cls)
    assert sum(v.numel() for v in sd.values()) == sum(p.numel() for p in m.parameters())
    w = sd["blocks.3.attn.qkv.weight"]
    assert abs(w.std().item() - 0.02) < 2e-3 and w.abs().max().item() <= 2.0 + 1e-6


def test_shard_indices_cover_everything_once():
    pl = load_pkg("pipeline")
    for n, world in [(10, 1), (10, 3), (50_000, 8), (5, 8)]:
        parts = [pl.shard_indices(n, r, world) for r in range(world)]
        flat = sorted(i for p in parts for i in p)
        assert flat == list(range(n))
        assert max(len(p) for p in parts) - min(len(p) for p in parts) <= 1
    with pytest.raises(ValueError):
        pl.shard_indices(10, 3, 2)


def test_synthetic_inputs_are_seeded():
    synth = load_pkg("synth")
    a, b = synth.blobs_image(64, 80, 5), synth.blobs_image(64, 80, 5)
    assert torch.equal(a, b) and a.dtype == torch.uint8 and tuple(a.shape) == (64, 80, 3)
    assert not torch.equal(a, synth.blobs_image(64, 80, 6))
    shapes = synth.voc_shapes(1000, 0)
    assert shapes == synth.voc_shapes(1000, 0) and max(max(s) for s in shapes) == 500
    f = synth.structured_features(100, 32, 4, 1)
    assert torch.equal(f, synth.structured_features(100, 32, 4, 1)) and f.dtype == torch.float32


def test_gemm_gelu_erf_constants():
    """The fc1 epilogue evaluates the exact-erf GELU as relu(x) - |x| 2^P(min(|x| / sqrt 2, c)) (csrc/common.cuh,
    gelu_erf). Emulate that float32 arithmetic with the constants parsed out of the kernel source against torch's
    erf GELU in float64 over the whole range fp16 activations can take."""
    import re
    src = (ROOT / "deep-spectral-segmentation_b200" / "csrc" / "common.cuh").read_text()
    coef = [np.float32(float(v)) for v in re.findall(r"#define DSS_GELU_P\d (-?[\d.e+-]+)f", src)]
    clamp = np.float32(float(re.search(r"#define DSS_GELU_CLAMP ([\d.]+)f", src).group(1)))
    assert len(coef) == 5, coef                            # p0 .. p4 of P(u) = sum p_k u^k
    x = np.concatenate([np.linspace(-12.0, 12.0, 480001), np.linspace(-6.0e4, 6.0e4, 20001)]).astype(np.float32)
    na = -np.abs(x)
    u = np.minimum((na * np.float32(-0.7071067811865476)).astype(np.float32), clamp)
    p = np.full_like(u, coef[4])
    for k in range(3, -1, -1):
        p = (p.astype(np.float64) * u.astype(np.float64) + np.float64(coef[k])).astype(np.float32)   # one rounding = fma
    q = np.exp2(p.astype(np.float64))
    q = (q * (1.0 + 2.4e-7)).astype(np.float32)            # ex2.approx: 2 ulp
    got = (na.astype(np.float64) * q.astype(np.float64) + np.maximum(x, np.float32(0)).astype(np.float64)).astype(np.float32)
    ref = torch.nn.functional.gelu(torch.from_numpy(x.astype(np.float64))).numpy()
    err = np.abs(got.astype(np.float64) - ref)
    assert err.max() < 8e-6, err.max()
    neg = (x < -1) & (x > -3)                               # relative accuracy down to -3 (values >= 4e-3; beyond that the
    assert np.all(err[neg] <= 2e-3 * np.abs(ref[neg]))      # 6e-6 absolute bound is below the fp16 normal range)


def test_batch_assembler_groups_by_shape_and_delivers_every_image_once(tmp_path):
    """io_pipeline.BatchAssembler (the decode side of extract_all): three image shapes, decode threads writing straight
    into the batches, only two batches per shape so that workers must wait for release(); every file has to come out
    exactly once, in a batch of its own shape, with the pixels cv2.imread + BGR->RGB gives (extract_utils.py:30-31)."""
    import cv2
    iop = load_pkg("io_pipeline"); utils = load_pkg("extract_utils")
    rng = np.random.default_rng(0)
    shapes = [(32, 48), (48, 32), (40, 40)]
    names = []
    for i in range(157):
        H, W = shapes[i % 3 if i < 150 else 2]
        name = f"im{i:04d}.png"
        cv2.imwrite(str(tmp_path / name), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        names.append(name)
    ds = utils.ImagesDataset(names, str(tmp_path))
    asm = iop.BatchAssembler(ds.load_raw, range(len(ds)), capacity=16, num_workers=5, slots=2)
    seen = {}
    held = []
    for b in asm:
        assert 1 <= b.assigned <= 16 and b.filled == b.assigned and len(b.items) == b.assigned
        for row, (path, index) in enumerate(b.items):
            assert index not in seen
            seen[index] = (b.key, b.host[row].clone())
        held.append(b)
        if len(held) > 1:            # like extract_all: a batch is given back one batch later
            asm.release(held.pop(0))
    assert sorted(seen) == list(range(len(ds)))
    for index, (key, pixels) in seen.items():
        want, path, idx = ds[index]
        assert idx == index and key == tuple(want.shape[:2])
        assert torch.equal(pixels, want)
    # an unreadable file surfaces as an exception in the consumer, not as a hang
    (tmp_path / "broken.png").write_bytes(b"not an image")
    bad = utils.ImagesDataset(names[:8] + ["broken.png"], str(tmp_path))
    with pytest.raises(IOError):
        for b in iop.BatchAssembler(bad.load_raw, range(len(bad)), capacity=4, num_workers=3):
            pass


def test_process_writer_splits_a_batch_into_row_ranges(tmp_path):
    """ProcessWriter.submit_batch sends each writer only its rows; the files must hold the row of their own image."""
    iop = load_pkg("io_pipeline")
    arrays = {"v": np.arange(10 * 3, dtype=np.float32).reshape(10, 3)}
    items = [(str(tmp_path / f"f{j}.pth"), j, {"id": f"f{j}"}, {"row": ("slice", "v"), "n": ("tensor0d", j)})
             for j in range(10) if j != 4]
    sent = []

    class Fake(iop.ProcessWriter):
        def __init__(self):
            self.procs = [None] * 3; self.submitted = 0; self.done = 0
            self.q = type("Q", (), {"put": lambda self_, m: sent.append(m)})()

        def _check(self):
            pass
    Fake().submit_batch(arrays, items)
    got = {}
    for arrs, part in sent:
        for path, j, extra, fields in part:
            got[extra["id"]] = iop._materialise(arrs, j, extra, fields)
    assert sorted(got) == sorted(f"f{j}" for j in range(10) if j != 4)
    for name, d in got.items():
        j = int(name[1:])
        assert torch.equal(d["row"], torch.from_numpy(arrays["v"][j])) and int(d["n"]) == j
    assert sum(a["v"].shape[0] for a, _ in sent) <= 10


def test_available_cpus_respects_affinity_and_quota(monkeypatch):
    """io_pipeline.available_cpus (pool sizing): never more than the affinity mask, at least 1, and the decode-thread
    default leaves room for the GPU-feeding thread and the writers."""
    import os
    iop = load_pkg("io_pipeline")
    n = iop.available_cpus()
    assert 1 <= n <= (os.cpu_count() or 1)
    if hasattr(os, "sched_getaffinity"):
        assert n <= len(os.sched_getaffinity(0))
    monkeypatch.delenv("DSS_IO_DECODE_THREADS", raising=False)
    w = iop.default_workers()
    assert 1 <= w <= max(1, n - 1) and w <= 32
    monkeypatch.setenv("DSS_IO_DECODE_THREADS", "5")
    assert iop.default_workers() == 5


def test_cli_commands_shard_their_work_list_by_rank(monkeypatch):
    """extract._my_share: under torchrun (RANK / WORLD_SIZE) every command takes the strided share of its sorted work
    list; the shares partition the list, a single process keeps everything, a rank outside the world is an error."""
    ex = load_pkg("extract")
    items = list(range(23))
    monkeypatch.delenv("RANK", raising=False); monkeypatch.delenv("WORLD_SIZE", raising=False)
    assert ex._my_share(items) == items and ex._rank_world() == (0, 1)
    seen = []
    for r in range(4):
        monkeypatch.setenv("RANK", str(r)); monkeypatch.setenv("WORLD_SIZE", "4")
        share = ex._my_share(items)
        assert share == items[r::4]
        seen += share
    assert sorted(seen) == items
    monkeypatch.setenv("RANK", "4")
    with pytest.raises(ValueError):
        ex._rank_world()


def test_batch_assembler_closes_partial_batches_under_memory_pressure(tmp_path):
    """Many shapes, few images each (the VOC situation): with max_pending small the assembler has to hand over partly
    filled batches early (largest first) instead of holding one open batch per shape; nothing may be lost or doubled."""
    import cv2
    iop = load_pkg("io_pipeline"); utils = load_pkg("extract_utils")
    rng = np.random.default_rng(1)
    names = []
    for i in range(120):
        H, W = 16 + 8 * (i % 7), 24 + 8 * ((i // 7) % 5)       # 35 distinct shapes
        name = f"v{i:04d}.png"
        cv2.imwrite(str(tmp_path / name), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        names.append(name)
    ds = utils.ImagesDataset(names, str(tmp_path))
    asm = iop.BatchAssembler(ds.load_raw, range(len(ds)), capacity=64, num_workers=4, slots=2, max_pending=8,
                             full_size_shapes=3, small_capacity=4)
    seen, sizes = set(), []
    for b in asm:
        assert b.assigned <= b.capacity and b.filled == b.assigned
        for row, (path, index) in enumerate(b.items):
            assert index not in seen
            seen.add(index)
            want = ds[index][0]
            assert tuple(want.shape[:2]) == b.key and torch.equal(b.host[row], want)
        sizes.append(b.assigned)
        asm.release(b)
    assert seen == set(range(len(ds)))
    assert max(sizes) < 64          # pressure closed the batches long before they were full
