"""CPU suite for Pillow's bilinear resize (resize.py, csrc/resize.cu) and extract_all's extract_eigs options: the
host-built window and weight tables, the fixed-point two-pass restatement against PIL.Image.resize itself, the RGB-file
check of colour mode, and the argument refusals of the C entry point, the Python wrapper, extract_all, extract_eigs and
_extract_eig, all raised before any device work."""

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import load_pkg

ONE = 1 << 22


def _pairs():
    """(H, W, H_out, W_out): every VOC shape at factors 16 and 8 of its 16-pixel crop (and 4 of its 8-pixel crop), the
    patch grids themselves, 1-pixel and same-size outputs, odd ratios and a few hundred random pairs."""
    synth = load_pkg("synth")
    pairs = []
    for (H, W), _ in synth.VOC_SHAPES:
        for P, f in ((16, 16), (16, 8), (8, 4), (8, 8)):
            pairs.append((H, W, H // P * P // f, W // P * P // f))
    pairs += [(1, 1, 1, 1), (7, 5, 7, 5), (31, 17, 1, 1), (31, 17, 31, 1), (31, 17, 1, 17), (100, 3, 9, 2),
              (97, 89, 13, 11), (64, 64, 63, 63), (65, 33, 64, 32), (301, 299, 37, 41), (500, 375, 499, 374)]
    rng = np.random.default_rng(1)
    for _ in range(300):
        H, W = (int(v) for v in rng.integers(1, 140, 2))
        pairs.append((H, W, int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))))
    return pairs


def test_tables_windows_and_weights():
    rz = load_pkg("resize")
    sizes = {(H, h) for H, W, h, w in _pairs()} | {(W, w) for H, W, h, w in _pairs()}
    for n_in, n_out in sorted(sizes):
        bounds, weights = rz.coeffs(n_in, n_out)
        taps = weights.shape[1]
        scale = n_in / n_out
        assert bounds.dtype == np.int32 and weights.dtype == np.int32 and bounds.shape == (n_out, 2)
        assert taps == 2 * int(np.ceil(max(scale, 1.0))) + 1
        first, count = bounds[:, 0], bounds[:, 1]
        assert (first >= 0).all() and (count >= 1).all() and (count <= taps).all() and (first + count <= n_in).all()
        assert (np.diff(first) >= 0).all()                                    # windows move with the output index
        for o in range(n_out):
            w = weights[o]
            assert (w[count[o]:] == 0).all() and (w >= 0).all()
            # normalised to 1 before rounding: the fixed-point sum is 2^22 up to half a unit per tap
            assert abs(int(w.sum()) - ONE) <= (count[o] + 1) // 2, (n_in, n_out, o, w)
            # the window holds every input pixel the widened triangle reaches, and only those
            centre, support = (o + 0.5) * scale, max(scale, 1.0)
            for x in (first[o] - 1, first[o] + count[o]):
                if 0 <= x < n_in:
                    assert abs(x + 0.5 - centre) >= support - 1e-9, (n_in, n_out, o, x)
            assert all(abs(x + 0.5 - centre) <= support + 0.5 for x in range(first[o], first[o] + count[o]))
        if n_in == n_out:                       # the identity: {1, 0} on each pixel, exact for every value
            assert (first == np.arange(n_in)).all() and (weights[:, 0] == ONE).all() and (weights[:, 1:] == 0).all()
        if n_out == 1:                          # one output pixel: the window is the whole input
            assert first[0] == 0 and count[0] == n_in


def test_fixed_point_restatement_equals_pillow():
    rz = load_pkg("resize")
    rng = np.random.default_rng(0)
    pairs = _pairs()
    assert len(pairs) > 300
    for H, W, h, w in pairs:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        want = np.array(Image.fromarray(img).resize((w, h), Image.BILINEAR))
        got = rz.resize_host(img, w, h)
        assert np.array_equal(got, want), (H, W, h, w)


def test_restatement_on_blobs_images_equals_pillow():
    """Smooth images with flat rectangles (the blobs recipe) reach the clipping and rounding edges differently from
    noise: every VOC shape at factors 16 and 8."""
    rz, synth = load_pkg("resize"), load_pkg("synth")
    for s, ((H, W), _) in enumerate(synth.VOC_SHAPES):
        img = synth.blobs_image(H, W, s).numpy()
        for f in (16, 8):
            h, w = H // 16 * 16 // f, W // 16 * 16 // f
            assert np.array_equal(rz.resize_host(img, w, h),
                                  np.array(Image.fromarray(img).resize((w, h), Image.BILINEAR))), (H, W, f)


def test_resize_entry_point_rejects_bad_arguments_before_any_device_work():
    _lib, rz = load_pkg("_lib"), load_pkg("resize")
    lib = _lib.load()
    n0 = lib.dss_kernel_launch_count()
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    by, wy = rz.coeffs(40, 10)
    bx, wx = rz.coeffs(30, 6)
    ty, tx = wy.shape[1], wx.shape[1]
    ws = int(lib.dss_resize_workspace_bytes(10, 6, ty, tx))
    assert 0 < ws <= (1 << 15)
    assert lib.dss_resize_workspace_bytes(0, 6, ty, tx) == 0

    def call(images=p, B=1, H=40, W=30, h=10, w=6, by_=by, wy_=wy, ty_=ty, bx_=bx, wx_=wx, tx_=tx, kind=0, out=p, ws_=p,
             ws_bytes=ws):
        ptr = lambda a: None if a is None else a.ctypes.data   # noqa: E731
        return lib.dss_resize_bilinear(images, B, H, W, h, w, ptr(by_), ptr(wy_), ty_, ptr(bx_), ptr(wx_), tx_, kind, out,
                                       ws_, ws_bytes, None)
    assert call(images=None) == -1
    assert call(out=None) == -1
    assert call(ws_=None) == -1
    assert call(by_=None) == -1
    assert call(wx_=None) == -1
    assert call(B=0) == -1
    assert call(h=0) == -1
    assert call(ty_=0) == -1
    assert call(h=41) == -1                   # upscaling
    assert call(w=31) == -1
    assert call(kind=2) == -1
    assert call(ws_bytes=ws - 1) == -3
    assert call(B=65536) == -4
    bad = by.copy()
    bad[3, 0] = 39                            # window past the input
    assert call(by_=bad) == -1
    bad = bx.copy()
    bad[0, 1] = tx + 1                        # more taps than the table holds
    assert call(bx_=bad) == -1
    bad = wx.copy()
    bad[1, 0] = -5
    assert call(wx_=bad) == -1
    assert call(H=39) == -1                   # tables built for 40 rows read row 39 + ... past a 39-row image
    msg = lib.dss_last_error().decode()
    assert "vertical window" in msg
    assert lib.dss_kernel_launch_count() == n0


def test_resize_wrapper_rejects_bad_images_before_any_device_work():
    _lib, rz = load_pkg("_lib"), load_pkg("resize")
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="image 1 is not a 3-channel"):
        rz.resize([torch.zeros(8, 8, 3, dtype=torch.uint8), torch.zeros(8, 8, dtype=torch.uint8)], 4, 4)
    with pytest.raises(ValueError, match="image 2 is \\(8, 9\\), image 0 is \\(8, 8\\)"):
        rz.resize([torch.zeros(8, 8, 3, dtype=torch.uint8)] * 2 + [torch.zeros(8, 9, 3, dtype=torch.uint8)], 4, 4)
    with pytest.raises(ValueError, match="3-channel"):
        rz.resize(torch.zeros(2, 8, 8, 4, dtype=torch.uint8), 4, 4)
    with pytest.raises(ValueError, match="uint8"):
        rz.resize(torch.zeros(2, 8, 8, 3), 4, 4)
    with pytest.raises(ValueError, match="no larger than the input"):
        rz.resize(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), 9, 4)
    with pytest.raises(ValueError, match="unknown output kind"):
        rz.resize(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), 4, 4, kind="f16")
    with pytest.raises(_lib.DssError, match="CUDA tensor"):
        rz.resize(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), 4, 4)
    assert _lib.launch_count() == n0


def _jpeg(path, img, mode=None):
    im = Image.fromarray(img) if mode is None else Image.fromarray(img).convert(mode)
    im.save(path, quality=92)
    return path


def test_colour_mode_reader_refuses_files_that_are_not_rgb(tmp_path):
    utils, synth = load_pkg("extract_utils"), load_pkg("synth")
    img = synth.blobs_image(48, 40, 3).numpy()
    rgb = _jpeg(tmp_path / "rgb.jpg", img)
    pixels, is_bgr = utils.read_image_raw_rgb_file(rgb)
    want, want_bgr = utils.read_image_raw(rgb)
    assert is_bgr == want_bgr and np.array_equal(pixels, want)
    for mode in ("L", "CMYK"):
        path = _jpeg(tmp_path / f"{mode}.jpg", img, mode)
        with pytest.raises(ValueError, match=f"{mode}.jpg: colour affinities need a 3-channel RGB image.*'{mode}'"):
            utils.read_image_raw_rgb_file(path)
        # the route it replaces fails on the same files
        lr = np.array(Image.open(path).resize((5, 6), Image.BILINEAR))
        with pytest.raises(ValueError):
            lr.reshape(1, 30, 3)


EIGS_OPTION_REFUSALS = [        # extract_eigs' options: refused by every command that runs the eigen stage
    (dict(which_matrix="affinity_torch"), RuntimeError, "torch.eig"),
    (dict(which_matrix="nope"), ValueError, "unknown which_matrix"),
    (dict(image_color_lambda=10.0, which_color_matrix="nope"), ValueError, "unknown which_color_matrix"),
    (dict(image_downsample_factor=0), ValueError, "positive integer"),
    (dict(image_downsample_factor=-8), ValueError, "positive integer"),
]
EXTRACT_ALL_REFUSALS = [
    (dict(image_downsample_factor=8, single_region_dir="S"), ValueError, "single_region_dir: .* cannot reshape"),
    (dict(image_downsample_factor=4, multi_region_dir="M"), ValueError, "multi_region_dir: .* twice as fine"),
    (dict(image_downsample_factor=12, multi_region_dir="M"), ValueError, "multi_region_dir"),
    (dict(model_name="resnet50"), ValueError, "Cannot get model"),
]


@pytest.mark.parametrize("command, kw, err, match",
                         [(c, *row) for c in ("extract_all", "extract_eigs", "_extract_eig") for row in EIGS_OPTION_REFUSALS]
                         + [("extract_all", *row) for row in EXTRACT_ALL_REFUSALS])
def test_extract_all_refuses_before_any_device_work(tmp_path, command, kw, err, match):
    """extract_all, extract_eigs and _extract_eig refuse unsupported options before any file or device work: no kernel
    launch, no output directory."""
    ex, _lib, iop = load_pkg("extract"), load_pkg("_lib"), load_pkg("io_pipeline")
    out = str(tmp_path / "eigs")
    features = tmp_path / "features"
    features.mkdir()
    (path, j, extra, fields), = ex._feature_files(str(features), [("a.jpg", 0, 64, 48)], [(0, 12)], "dino_vits16", 16)
    torch.save(iop._materialise({"k": np.ones((12, 384), np.float32)}, j, extra, fields), path)
    n0 = _lib.launch_count()
    if command == "extract_all":
        args, kwargs = (), dict(images_list=str(tmp_path / "missing.txt"), images_root=str(tmp_path),
                                model_name="dino_vits16", features_dir=None, eigs_dir=out)
        kwargs.update(kw)
        for key in ("single_region_dir", "multi_region_dir"):
            if key in kwargs:
                kwargs[key] = str(tmp_path / kwargs[key])
    elif command == "extract_eigs":
        args, kwargs = (str(tmp_path), str(features), out), dict(K=4, **kw)
    else:
        args, kwargs = ((0, path), 4, str(tmp_path), out), kw
    with pytest.raises(err, match=match):
        getattr(ex, command)(*args, **kwargs)
    assert _lib.launch_count() == n0
    assert not (tmp_path / "eigs").exists()      # refused before any output directory is made


def test_eig_options_accept_the_grids_the_segmentation_commands_read():
    """The patch grid, the grid twice as fine with multi_region_dir, and the affinity modes (their eigenvectors are on
    the patch grid whatever the factor) pass the option checks; the grid is the patch size divided by the factor."""
    ex, vit = load_pkg("extract"), load_pkg("vit")

    def check(model_name, which_matrix, factor, lam, which_color_matrix, single_region, multi_region):
        """-> (Laplacian mode, colour terms, factor) of options that pass every check."""
        opts = ex._EigOptions(K=20, which_matrix=which_matrix, which_color_matrix=which_color_matrix, normalize=True,
                              threshold_at_zero=True, lapnorm=True, image_downsample_factor=factor,
                              image_color_lambda=lam)
        ex._extract_all_options(model_name, opts, single_region, multi_region)
        return opts.laplacian, opts.colour, opts.factor(vit.arch(model_name)[0])

    assert check("dino_vits16", "laplacian", None, 0.0, "knn", True, True) == (True, False, 16)
    assert check("dino_vits16", "laplacian", 16, 10.0, "rw", True, True) == (True, True, 16)
    assert check("dino_vits16", "laplacian", 8, 10.0, "knn", False, True) == (True, True, 8)
    assert check("dino_vits8", "matting_laplacian", 4, 0.0, "knn", False, True) == (True, False, 4)
    assert check("dino_vits16", "laplacian", 4, 0.0, "knn", False, False) == (True, False, 4)
    assert check("dino_vits16", "affinity", 8, 10.0, "rw", True, True) == (False, False, 16)
    assert check("dino_vits16", "affinity_svd", 3, 10.0, "knn", True, True) == (False, False, 16)


def test_cli_parses_the_new_options():
    ex, cli = load_pkg("extract"), load_pkg("cli")
    args, kwargs = cli.parse_args(ex.extract_all, ["l.txt", "root", "dino_vits16", "f", "e", "--image_downsample_factor",
                                                   "8", "--which_matrix", "affinity"])
    assert args == ["l.txt", "root", "dino_vits16", "f", "e"]
    assert kwargs == {"image_downsample_factor": 8, "which_matrix": "affinity"}
