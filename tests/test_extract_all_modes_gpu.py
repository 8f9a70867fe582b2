"""GPU suite for extract_eigs' options in extract_all and the device resize behind its colour affinities.

- resize.resize equals PIL.Image.resize(BILINEAR) bit for bit: uint8 on a few hundred size pairs (every VOC shape at
  factors 16 and 8 among them), and fp32 / uint8 against extract_eigs' host route (_color_inputs) on JPEG files.
- For every new mode, at batch sizes 1 and 4 over mixed shapes, extract_all writes feature, eigs and PNG files equal to
  extract_features + extract_eigs (+ the segmentation commands on extract_all's own files): torch.equal on every
  tensor, byte equality on every PNG.
- Colour mode never calls the host route, and refuses files that are not RGB by name."""
import numpy as np
import pytest
import torch
from PIL import Image

from conftest import load_pkg
from test_cpu_resize import _pairs

pytestmark = pytest.mark.gpu


def test_device_resize_equals_pillow(cuda):
    rz = load_pkg("resize")
    rng = np.random.default_rng(2)
    for H, W, h, w in _pairs():
        imgs = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
        got = rz.resize(torch.from_numpy(imgs).to(cuda), h, w, "u8").cpu().numpy()
        got_f = rz.resize(torch.from_numpy(imgs).to(cuda), h, w, "f32").cpu().numpy()
        for b in range(3):
            want = np.array(Image.fromarray(imgs[b]).resize((w, h), Image.BILINEAR)).reshape(h * w, 3)
            assert np.array_equal(got[b], want), (H, W, h, w, b)
            assert np.array_equal(got_f[b], (want / 255.0).astype(np.float32)), (H, W, h, w, b)


def test_device_resize_equals_the_host_colour_route(cuda, tmp_path):
    """The inputs extract_eigs builds from the JPEG files (_color_inputs: PIL open + resize, /255 in float64 then fp32
    for 'knn', uint8 for 'rw') equal the device resize of the decoded images extract_all has on the GPU."""
    ex, rz, synth, utils = load_pkg("extract"), load_pkg("resize"), load_pkg("synth"), load_pkg("extract_utils")
    shapes = [hw for hw, _ in synth.VOC_SHAPES] + [(97, 131), (64, 48), (17, 33)]
    for s, (H, W) in enumerate(shapes):
        ids = []
        for j in range(2):
            ids.append(f"im{s}_{j}")
            Image.fromarray(synth.blobs_image(H, W, 10 * s + j).numpy()).save(tmp_path / f"{ids[-1]}.jpg", quality=90)
        dec = torch.stack([torch.from_numpy(np.ascontiguousarray(utils.read_image_rgb(tmp_path / f"{i}.jpg")))
                           for i in ids]).to(cuda)
        for f in (16, 8, 4):
            h, w = H // 16 * 16 // f, W // 16 * 16 // f
            if h == 0 or w == 0:
                continue
            for kind, matrix in (("f32", "knn"), ("u8", "rw")):
                want = ex._color_inputs(str(tmp_path), ids, w, h, matrix, cuda)
                got = rz.resize(dec, h, w, kind)
                assert got.dtype == want.dtype and torch.equal(got, want), (H, W, f, kind)


# ---------------------------------------------------------------------------------------------------------------
SHAPES = {"dino_vits16": [(160, 208), (224, 160), (176, 176)], "dino_vits8": [(96, 128), (128, 96), (112, 112)]}
K = 6
# (id, model, options, single-region PNGs, multi-region PNGs, adaptive cluster counts)
MODES = [
    ("factor8", "dino_vits16", dict(image_downsample_factor=8), False, True, False),
    ("factor16", "dino_vits16", dict(image_downsample_factor=16), True, True, False),
    ("vits8_factor4", "dino_vits8", dict(image_downsample_factor=4), False, True, False),
    ("affinity", "dino_vits16", dict(which_matrix="affinity"), True, True, True),
    ("affinity_svd", "dino_vits16", dict(which_matrix="affinity_svd"), True, True, False),
    ("knn", "dino_vits16", dict(image_color_lambda=10.0, which_color_matrix="knn"), True, True, False),
    ("knn_factor8", "dino_vits16", dict(image_color_lambda=10.0, which_color_matrix="knn", image_downsample_factor=8),
     False, True, False),
    ("rw", "dino_vits16", dict(image_color_lambda=10.0, which_color_matrix="rw"), True, True, False),
    ("rw_factor8", "dino_vits16", dict(image_color_lambda=10.0, which_color_matrix="rw", image_downsample_factor=8),
     False, True, False),
]


def _write_images(root, model):
    synth = load_pkg("synth")
    root.mkdir(parents=True, exist_ok=True)
    names = []
    for s, (H, W) in enumerate(SHAPES[model]):
        for j in range(2):       # two images per shape, interleaved so that batches of 4 mix shapes in the list
            names.append(f"im{j}{s}.jpg")
            Image.fromarray(synth.blobs_image(H, W, 7 * s + j).numpy()).save(root / names[-1], quality=95)
    return sorted(names)


def _assert_same_pth(a, b, what):
    da, db = torch.load(a, weights_only=False), torch.load(b, weights_only=False)
    assert sorted(da) == sorted(db), what
    for key in da:
        x, y = da[key], db[key]
        if isinstance(x, np.ndarray):
            assert isinstance(y, np.ndarray) and x.dtype == y.dtype and np.array_equal(x, y), (what, key)
        elif isinstance(x, torch.Tensor):
            assert x.dtype == y.dtype and torch.equal(x, y), (what, key)
        else:
            assert x == y, (what, key)


@pytest.mark.parametrize("mode, model, opts, single, multi, adaptive", MODES, ids=[m[0] for m in MODES])
def test_extract_all_mode_equals_the_file_based_commands(cuda, tmp_path, mode, model, opts, single, multi, adaptive):
    ex = load_pkg("extract")
    root = tmp_path / "images"
    names = _write_images(root, model)
    lst = tmp_path / "list.txt"
    lst.write_text("\n".join(names) + "\n")
    # the file-based route: features, then eigs
    ex.extract_features(str(lst), str(root), model, 4, str(tmp_path / "f_ref"), seed=0)
    ex.extract_eigs(str(root), str(tmp_path / "f_ref"), str(tmp_path / "e_ref"), K=K, **opts)
    seg = dict(non_adaptive_num_segments=3, adaptive=adaptive)
    for bs in (1, 4):
        d = {n: tmp_path / f"{n}{bs}" for n in ("f", "e", "s", "m")}
        ex.extract_all(str(lst), str(root), model, str(d["f"]), str(d["e"]), K=K, batch_size=bs, seed=0,
                       single_region_dir=str(d["s"]) if single else None,
                       multi_region_dir=str(d["m"]) if multi else None, **seg, **opts)
        for n in names:
            stem = n[:-4]
            _assert_same_pth(d["f"] / f"{stem}.pth", tmp_path / "f_ref" / f"{stem}.pth", (mode, bs, "features", stem))
            _assert_same_pth(d["e"] / f"{stem}.pth", tmp_path / "e_ref" / f"{stem}.pth", (mode, bs, "eigs", stem))
        # the segmentation commands on extract_all's own feature and eigs files
        if single:
            ex.extract_single_region_segmentations(str(d["f"]), str(d["e"]), str(tmp_path / f"s_ref{bs}"))
        if multi:
            ex.extract_multi_region_segmentations(str(d["f"]), str(d["e"]), str(tmp_path / f"m_ref{bs}"), **seg)
        for kind, on in (("s", single), ("m", multi)):
            if not on:
                continue
            for n in names:
                png = f"{n[:-4]}.png"
                assert (d[kind] / png).read_bytes() == (tmp_path / f"{kind}_ref{bs}" / png).read_bytes(), (mode, bs, kind, n)
        if multi and opts.get("image_downsample_factor") in (8, 4):      # half the patch size: the 2x finer grid
            P = 16 if model == "dino_vits16" else 8
            H, W = SHAPES[model][0]
            im = np.array(Image.open(d["m"] / "im00.png"))
            assert im.shape == (2 * (H // P), 2 * (W // P))


def test_extract_all_colour_mode_reads_each_image_once(cuda, tmp_path, monkeypatch):
    ex = load_pkg("extract")
    root = tmp_path / "images"
    names = _write_images(root, "dino_vits16")
    lst = tmp_path / "list.txt"
    lst.write_text("\n".join(names) + "\n")

    def host_route(*args, **kwargs):
        raise AssertionError("extract_all called the host colour route")
    monkeypatch.setattr(ex, "_color_inputs", host_route)
    monkeypatch.setattr(ex, "_load_image_lr_u8", host_route)
    for matrix in ("knn", "rw"):
        out = tmp_path / f"eigs_{matrix}"
        st = ex.extract_all(str(lst), str(root), "dino_vits16", None, str(out), K=K, batch_size=4, seed=0,
                            image_color_lambda=10.0, which_color_matrix=matrix, image_downsample_factor=8)
        assert st["images"] == len(names) and len(list(out.iterdir())) == len(names)


def test_extract_all_colour_mode_refuses_grayscale_files_by_name(cuda, tmp_path):
    ex, synth = load_pkg("extract"), load_pkg("synth")
    root = tmp_path / "images"
    root.mkdir()
    Image.fromarray(synth.blobs_image(64, 64, 0).numpy()).save(root / "a.jpg")
    Image.fromarray(synth.blobs_image(64, 64, 1).numpy()).convert("L").save(root / "b.jpg")
    (tmp_path / "list.txt").write_text("a.jpg\nb.jpg\n")
    with pytest.raises(ValueError, match="b.jpg: colour affinities need a 3-channel RGB image"):
        ex.extract_all(str(tmp_path / "list.txt"), str(root), "dino_vits16", None, str(tmp_path / "e"), K=4, seed=0,
                       image_color_lambda=10.0)
    # without colour terms the same list runs (the decoder makes 3 channels of the gray file, as extract_features does)
    ex.extract_all(str(tmp_path / "list.txt"), str(root), "dino_vits16", None, str(tmp_path / "e2"), K=4, seed=0)
    assert len(list((tmp_path / "e2").iterdir())) == 2
