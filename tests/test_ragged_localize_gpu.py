"""-m gpu: object localization on batches of mixed image sizes, bit for bit with the uniform calls on each image alone.

- dss_vit_forward_last_ragged: every image's q / k / v features and CLS-attention rows (pad 0 and 1) equal
  dss_vit_forward_last on that image alone, in both precision modes, for ViT-S/16 and ViT-B/8; the rows past N_b are +0.0
  although outputs and workspace start as NaN.
- The premise of ragged LOST: the N_b x N_b block of the un-normalised affinity of zero-padded features is the affinity
  of the image alone.
- dss_lost_boxes_ragged / dss_dinoseg_boxes_ragged: boxes, seeds and status equal the uniform call per image.
- localize.main writes the preds.pkl and results.txt the per-image uniform route gives, at several batch sizes."""
import pickle

import numpy as np
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

PRECISIONS = ("fp16", "fp32")
_MODELS = {}


def _model(name="dino_vits16", precision="fp16"):
    key = (name, precision)
    if key not in _MODELS:
        _MODELS[key] = load_pkg("vit").get_model(name, seed=0, device="cuda", precision=precision)[0]
    return _MODELS[key]


def _images(shapes, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g).cuda() for H, W in shapes]


def _is_pos_zero(x):
    return bool((x.contiguous().view(torch.int32) == 0).all())


def _ragged_last(model, ims, which, pad, n_max=None):
    """dss_vit_forward_last_ragged with outputs and workspace filled with NaN first."""
    L = load_pkg("_lib")
    vit = load_pkg("vit")
    packed, dims = model._ragged_args(ims, None)
    grids = vit.ragged_grids(dims.tolist(), model.patch_size, pad)
    n = max(g[0] for g in grids) if n_max is None else n_max
    ws = model._ragged_workspace(dims, L.VIT_RAGGED_PAD if pad else L.VIT_RAGGED_K)
    ws.fill_(0xFF)   # every float of the workspace a NaN
    B = len(ims)
    f = torch.full((B, n, model.dim), float("nan"), device="cuda")
    a = torch.full((B, model.num_heads, n), float("nan"), device="cuda")
    L.check(model.lib.dss_vit_forward_last_ragged(model._h, packed.data_ptr(), dims.data_ptr(), B, int(pad), which,
                                                  f.data_ptr(), n, a.data_ptr(), ws.data_ptr(), ws.numel(),
                                                  L.stream_ptr(model.device)), "dss_vit_forward_last_ragged")
    return f, a, grids


def _check_last(model, shapes, pads=(0, 1), whiches=(0, 1, 2), seed=0, n_extra=0):
    P = model.patch_size
    for pad in pads:
        keep = [s for s in shapes if pad or (s[0] >= P and s[1] >= P)]
        ims = _images(keep, seed)
        for which in whiches:
            n_max = max(g[0] for g in load_pkg("vit").ragged_grids(keep, P, pad)) + n_extra
            f, a, grids = _ragged_last(model, ims, which, pad, n_max)
            for b, (im, (N, gh, gw)) in enumerate(zip(ims, grids)):
                fa, aa = model.forward_last(im[None], "qkv"[which], pad=bool(pad), cls_attn=True)
                assert fa.shape[1] == N
                assert torch.equal(f[b, :N], fa[0]), (tuple(im.shape), pad, which)
                assert torch.equal(a[b, :, :N], aa[0]), (tuple(im.shape), pad, which)
                assert _is_pos_zero(f[b, N:]) and _is_pos_zero(a[b, :, N:]), (tuple(im.shape), pad, which)


def _edge_shapes(P):
    return [(P - 1, 3 * P), (1, 1), (P, P), (2 * P, 5 * P), (P * 3 + 1, P * 2 + 1),   # below P, multiples, P k + 1
            (P, 9 * P), (7 * P, P - 3),                                                  # 1 x n and n x 1 grids
            (P, 126 * P), (P, 127 * P - 5), (8 * P, 16 * P), (P + 1, 63 * P + 7)]          # N_b + 1 = 127, 128, 129


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_last_ragged_vits16(cuda, precision):
    _check_last(_model("dino_vits16", precision), _edge_shapes(16) + [(375, 500), (224, 224)])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_last_ragged_vitb8(cuda, precision):
    _check_last(_model("dino_vitb8", precision), _edge_shapes(8) + [(250, 170)], whiches=(1,), seed=1, n_extra=3)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_last_ragged_voc_mix(cuda, precision):
    synth = load_pkg("synth")
    rng = np.random.default_rng(5)
    shapes = synth.voc_shapes(48, seed=5) + [(500, int(w)) if i % 2 else (int(w), 500)
                                             for i, w in enumerate(rng.integers(90, 500, 16))]
    _check_last(_model("dino_vits16", precision), shapes, pads=(1,), whiches=(1,), seed=2)


def _rows(N, d, g, spread=True):
    x = torch.randn(N, d, generator=g, dtype=torch.float64)
    if spread:   # row norms from 1e-3 to 1e3
        norms = torch.logspace(-3, 3, N, dtype=torch.float64)[torch.randperm(N, generator=g)]
        x = x / x.norm(dim=1, keepdim=True) * norms[:, None]
    return x.float()


def test_affinity_of_zero_padded_features_is_the_solo_affinity(cuda):
    spectral = load_pkg("spectral")
    g = torch.Generator().manual_seed(7)
    for n_max in (129, 1024, 1025):
        Ns = [n for n in (1, 127, 128, 129, 768) if n <= n_max]
        feats = [_rows(n, 384, g) for n in Ns]
        padded = torch.zeros(len(Ns), n_max, 384)
        for b, x in enumerate(feats):
            padded[b, :x.shape[0]] = x
        A = spectral.affinity(padded.cuda(), normalize=False, threshold_at_zero=False, scale_by_max=False)
        for b, x in enumerate(feats):
            n = x.shape[0]
            solo = spectral.affinity(x[None].cuda(), normalize=False, threshold_at_zero=False, scale_by_max=False)
            assert torch.equal(A[b, :n, :n], solo[0, :n, :n]), (n, n_max)


def _lost_case(grids, seed, zero_seed_image=None, d=64):
    """Padded features [B, n_max, d] of clustered patches, zero rows past each grid; image zero_seed_image has one
    all-zero patch (degree 0: the seed, with no similar patch: status 2)."""
    synth = load_pkg("synth")
    n_max = max(gh * gw for gh, gw in grids)
    f = torch.zeros(len(grids), n_max, d)
    for b, (gh, gw) in enumerate(grids):
        x = synth.clustered_features(gh * gw, d, n_clusters=3, seed=seed + b)
        if b == zero_seed_image:
            x[(gh * gw) // 2] = 0
        f[b, :gh * gw] = x
    return f.cuda()


def _check_lost(grids, sizes, ks, seed, zero_seed_image=None, P=16):
    loc = load_pkg("localize")
    f = _lost_case(grids, seed, zero_seed_image)
    for k in ks:
        boxes, seeds, status = loc.lost_boxes_ragged(f, grids, sizes, P, k)
        for b, ((gh, gw), s) in enumerate(zip(grids, sizes)):
            ob, os_, ost = loc.lost_boxes(f[b:b + 1, :gh * gw].contiguous(), (gh, gw), s, P, k)
            assert (boxes[b].tolist(), int(seeds[b]), int(status[b])) == (ob[0].tolist(), int(os_[0]), int(ost[0])), \
                (b, gh, gw, k)
        if zero_seed_image is not None:
            assert status[zero_seed_image] == load_pkg("_lib").LOC_SEED_IN_BACKGROUND


def test_lost_boxes_ragged_equal_each_image_alone(cuda):
    grids = [(1, 1), (3, 5), (24, 32), (1, 40), (40, 1), (8, 16), (32, 32), (11, 13)]
    sizes = [(1 + 16 * (gh - 1) + 5, 16 * gw) for gh, gw in grids]
    _check_lost(grids, sizes, (1, 100, 2000), seed=3, zero_seed_image=5)


def test_dinoseg_boxes_ragged_equal_each_image_alone(cuda):
    loc = load_pkg("localize")
    grids = [(1, 1), (2, 2), (24, 32), (1, 40), (40, 1), (8, 16), (32, 32), (11, 13)]
    heads = 6
    _check_dinoseg(loc, grids, heads, seed=4)


def _check_dinoseg(loc, grids, heads, seed, P=16):
    g = torch.Generator().manual_seed(seed)
    n_max = max(gh * gw for gh, gw in grids)
    a = torch.zeros(len(grids), heads, n_max)
    for b, (gh, gw) in enumerate(grids):
        x = torch.rand(heads, gh * gw, generator=g) ** 4
        a[b, :, :gh * gw] = x / x.sum(dim=1, keepdim=True)
    a = a.cuda()
    boxes, status = loc.dinoseg_boxes_ragged(a, grids, P, heads - 1)
    for b, (gh, gw) in enumerate(grids):
        ob, ost = loc.dinoseg_boxes(a[b:b + 1, :, :gh * gw].contiguous(), (gh, gw), P, heads - 1)
        assert (boxes[b].tolist(), int(status[b])) == (ob[0].tolist(), int(ost[0])), (b, gh, gw)


def test_300_image_ragged_batch(cuda):
    loc = load_pkg("localize")
    rng = np.random.default_rng(11)
    grids = [(int(rng.integers(1, 33)), int(rng.integers(1, 33))) for _ in range(300)]
    sizes = [(16 * gh - int(rng.integers(0, 16)), 16 * gw - int(rng.integers(0, 16))) for gh, gw in grids]
    _check_lost(grids, sizes, (100,), seed=20, zero_seed_image=150)
    _check_dinoseg(loc, grids, 6, seed=21)


def test_boxes_from_a_ragged_forward(cuda):
    """The command's route on one mixed batch: ragged forward, padded affinity and ragged boxes against
    forward_last + lost_boxes / dinoseg_boxes on each image."""
    loc = load_pkg("localize")
    synth = load_pkg("synth")
    model = _model()
    shapes = [(333, 500), (15, 40), (224, 224), (500, 375), (97, 130), (16, 16)]
    ims = [synth.blobs_image(H, W, seed=30 + i).cuda() for i, (H, W) in enumerate(shapes)]
    f, a, grids = model.forward_last_ragged(ims, which="k", pad=True, cls_attn=True)
    lb, ls_, lst = loc.lost_boxes_ragged(f, [g[1:] for g in grids], shapes, 16, 100)
    db, dst = loc.dinoseg_boxes_ragged(a, [g[1:] for g in grids], 16, model.num_heads - 1)
    for b, (im, (N, gh, gw)) in enumerate(zip(ims, grids)):
        fa, aa = model.forward_last(im[None], "k", pad=True, cls_attn=True)
        ob, os_, ost = loc.lost_boxes(fa, (gh, gw), shapes[b], 16, 100)
        assert (lb[b].tolist(), int(ls_[b]), int(lst[b])) == (ob[0].tolist(), int(os_[0]), int(ost[0])), shapes[b]
        ob, ost = loc.dinoseg_boxes(aa, (gh, gw), 16, model.num_heads - 1)
        assert (db[b].tolist(), int(dst[b])) == (ob[0].tolist(), int(ost[0])), shapes[b]


# ------------------------------------------------------------------------------------------------ the command
_XML = ("<annotation><filename>{name}.jpg</filename><size><width>{W}</width><height>{H}</height><depth>3</depth>"
        "</size><object><name>cat</name><truncated>0</truncated><difficult>0</difficult><bndbox><xmin>{x0}</xmin>"
        "<ymin>{y0}</ymin><xmax>{x1}</xmax><ymax>{y1}</ymax></bndbox></object></annotation>")


def _uniform_route(model, img, method):
    loc = load_pkg("localize")
    P = model.patch_size
    H, W = img.shape[:2]
    x = torch.tensor(img)[None].cuda()
    grid = (-(-H // P), -(-W // P))
    if method == "dinoseg":
        _, a = model.forward_last(x, "k", pad=True, feats=False, cls_attn=True)
        boxes, status = loc.dinoseg_boxes(a, grid, P, 4)
    else:
        f, _ = model.forward_last(x, "k", pad=True)
        boxes, _, status = loc.lost_boxes(f, grid, (H, W), P, 100)
    return boxes[0], int(status[0])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("method", ["lost", "dinoseg"])
def test_main_writes_the_per_image_route(cuda, tmp_path, precision, method):
    from PIL import Image
    loc = load_pkg("localize")
    synth = load_pkg("synth")
    model = _model("dino_vits16", precision)
    rng = np.random.default_rng(17)
    shapes = synth.voc_shapes(14, seed=17) + [(500, 200), (120, 500), (40, 30), (281, 500), (500, 500), (10, 500)]
    voc = tmp_path / "VOC2007" / "VOCdevkit" / "VOC2007"
    for sub in ("Annotations", "JPEGImages", "ImageSets/Main"):
        (voc / sub).mkdir(parents=True)
    ids, want = [], {}
    for i, (H, W) in enumerate(shapes):
        name = f"{i:06d}"
        img = synth.blobs_image(H, W, seed=100 + i).numpy()
        Image.fromarray(img).save(voc / "JPEGImages" / f"{name}.jpg", quality=95)
        decoded = loc.load_rgb(voc / "JPEGImages" / f"{name}.jpg")
        box, status = _uniform_route(model, decoded, method)
        if status != 0:   # the command raises for such an image, as the reference does; keep the tree runnable
            continue
        x0, y0 = int(rng.integers(1, W // 2 + 1)), int(rng.integers(1, H // 2 + 1))
        x1, y1 = int(rng.integers(x0, W + 1)), int(rng.integers(y0, H + 1))
        (voc / "Annotations" / f"{name}.xml").write_text(_XML.format(name=name, H=H, W=W, x0=x0, y0=y0, x1=x1, y1=y1))
        ids.append(name)
        want[f"{name}.jpg"] = box
    assert len(ids) >= 12
    (voc / "ImageSets" / "Main" / "trainval.txt").write_text("".join(f"{i}\n" for i in ids))
    gt = {n: loc.extract_gt_voc(loc.parse_voc_xml(voc / "Annotations" / f"{n[:-4]}.xml"))[0] for n in want}
    hits = sum(loc.corloc_hit(want[n], gt[n]) for n in want)
    results = ("corloc,%.1f,,\n" % (100 * hits / len(want))).encode()
    for bs in (1, 7, 64):
        out = tmp_path / f"out{bs}"
        argv = ["--dataset_root", str(tmp_path / "VOC2007"), "--output_dir", str(out), "--seed", "0",
                "--precision", precision, "--batch_size", str(bs)] + (["--dinoseg"] if method == "dinoseg" else [])
        loc.main(argv)
        folder = out / "VOC07_trainval" / loc.experiment_name(loc.parse_args(argv))
        preds = pickle.loads((folder / "preds.pkl").read_bytes())
        assert list(preds) == list(want)
        for n in want:
            assert preds[n].dtype == np.int64 and np.array_equal(preds[n], want[n]), (bs, n)
        assert (folder / "results.txt").read_bytes() == results
