"""CPU suite for the dense CRF: the label upsampling restatement against cv2, the float64 lattice against the exact
Gaussian filter, the oracle against the reference's stored outputs (and the reference itself when present), the host
label-map rules, and argument checks of the new C entry points."""
import sys

import numpy as np
import pytest

from conftest import ROOT, load_pkg

GOLDEN = ROOT / "tests" / "golden"
CASES = sorted(p.stem[len("ref_crf_"):] for p in GOLDEN.glob("ref_crf_*.npz"))

# Measured on the seeded 64 x 64 blobs images below (float64 lattice vs exact dense sums, symmetric normalisation):
#   max |lattice - exact| / max |exact| per filter: bilateral 0.21 .. 0.39, spatial 0.034 .. 0.041
#   mean-field labels (5 iterations, unary_eps 0.2, 4 classes) equal to the exact filter's: 96.7 .. 98.1 % of pixels
LATTICE_REL_ERR = {5: 0.5, 2: 0.06}
LABEL_AGREEMENT = 0.95


def _golden(name):
    return np.load(GOLDEN / f"ref_crf_{name}.npz", allow_pickle=False)


def _blobs(H, W, seed):
    return load_pkg("synth").blobs_image(H, W, seed).numpy()


@pytest.mark.parametrize("P", [16, 8, 14])
def test_label_upsampling_equals_cv2(P):
    cv2 = pytest.importorskip("cv2")
    from oracle import crf_ref
    crf = load_pkg("crf")
    rng = np.random.default_rng(P)
    for H, W in [(P, P), (P + 1, 2 * P - 1), (37, 45), (100, 97), (375, 500), (500, 333), (281, 500)]:
        if H < P or W < P:
            continue
        for sh, sw in [(H // P, W // P), (H // P + 1, W // P), (3, 5), (H // P + 2, W // P + 3)]:
            seg = rng.integers(0, 255, (sh, sw)).astype(np.uint8)
            Hp, Wp = H // P * P, W // P * P
            ref = cv2.resize(seg, dsize=(W, H), interpolation=cv2.INTER_NEAREST)
            ref[:Hp, :Wp] = cv2.resize(seg, dsize=(Wp, Hp), interpolation=cv2.INTER_NEAREST)
            assert np.array_equal(crf_ref.upsample_labels(seg, H, W, P), ref), (H, W, sh, sw)
            assert crf.full_resolution_values(seg, H, W, P) == set(np.unique(ref).tolist())


def test_prepare_segmap_binary_rule_and_label_range():
    crf = load_pkg("crf")
    m = np.array([[0, 255], [255, 0]], np.uint8)
    assert np.array_equal(crf.prepare_segmap(m, 32, 32, 16, 2), [[0, 1], [1, 0]])
    only = np.full((2, 2), 255, np.uint8)   # {255} alone is not {0, 255}: kept, and 255 >= num_classes
    with pytest.raises(ValueError, match="seg.png: label 255"):
        crf.prepare_segmap(only, 32, 32, 16, 21, "seg.png")
    three = np.array([[0, 1], [255, 0]], np.uint8)
    with pytest.raises(ValueError, match="label 255"):
        crf.prepare_segmap(three, 32, 32, 16, 21)
    with pytest.raises(ValueError, match="smaller than one"):
        crf.prepare_segmap(m, 15, 32, 16, 2)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_lattice_against_exact_filter(seed):
    from oracle import crf_ref
    img = _blobs(64, 64, 100 + seed)
    fb, fs = crf_ref.crf_features(img, 80, 13, 3)
    v = np.random.default_rng(seed).random((64 * 64, 4))
    for f in (fb, fs):
        lat = crf_ref.Lattice(f)
        a = lat.filter(v, True)
        e = crf_ref.exact_filter(f, v, True)
        rel = np.abs(a - e).max() / np.abs(e).max()
        assert rel < LATTICE_REL_ERR[f.shape[1]], (f.shape[1], rel)
        ones = lat.apply(np.ones((f.shape[0], 1)))
        assert (ones > 0).all()                     # L(1) > 0: every pixel's own splat comes back
        sub = np.eye(f.shape[0])[:, :256]
        K = lat.filter(sub, True)[:256]
        # n L n is symmetric up to the blur of missing neighbours at the lattice's edge (directions applied in turn):
        # ||K - K^T||_F / ||K||_F measured 0.11 on these 256 pixels of the image corner
        assert np.linalg.norm(K - K.T) < 0.2 * np.linalg.norm(K)
        assert np.abs(crf_ref.exact_filter(f, sub, True)[:256] - crf_ref.exact_filter(f, sub, True)[:256].T).max() < 1e-12


def test_mean_field_lattice_label_agreement_with_exact():
    from oracle import crf_ref
    worst = 1.0
    for seed in range(3):
        img = _blobs(64, 64, 100 + seed)
        seg = np.random.default_rng(seed).integers(0, 4, (8, 8)).astype(np.uint8)
        prob = np.eye(4)[crf_ref.upsample_labels(seg, 64, 64, 8)]
        _, l_lat, _ = crf_ref.mean_field(img, prob, (10, 80, 13, 3, 3, 5), 0.2)
        _, l_ex, _ = crf_ref.mean_field(img, prob, (10, 80, 13, 3, 3, 5), 0.2, filter="exact")
        worst = min(worst, float((l_lat == l_ex).mean()))
    assert worst >= LABEL_AGREEMENT, worst


def test_embedding_is_exact_on_lattice_points():
    """A point of the remainder-0 lattice has weight 1 on its own vertex; float64 keys are integers."""
    from oracle import crf_ref
    keys, w = crf_ref.embed(np.zeros((3, 5)))
    assert np.array_equal(w[:, 0], np.ones(3)) and np.abs(w[:, 1:]).max() == 0
    assert np.array_equal(keys[0, 0], np.zeros(5, np.int64))
    rng = np.random.default_rng(0)
    keys, w = crf_ref.embed(rng.normal(size=(1000, 2)) * 50)
    assert np.allclose(w.sum(1), 1.0) and (w > -1e-12).all()


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_fixtures(name):
    from oracle import crf_ref
    z = _golden(name)
    w1, alpha, beta, w2, gamma, it = z["params"].tolist()
    P, M = int(z["P"]), int(z["num_classes"])
    image = z["image"]
    H, W = image.shape[:2]
    crf = load_pkg("crf")
    seg = crf.prepare_segmap(z["segmap"], H, W, P, M)
    up = crf_ref.upsample_labels(seg, H, W, P)
    Qs, labels, counts = crf_ref.mean_field(image, np.eye(M)[up], (w1, alpha, beta, w2, gamma, it), float(z["unary_eps"]))
    assert np.array_equal(labels, z["labels"])
    assert np.abs(Qs[-1] - z["Q"]).max() < 1e-12
    assert tuple(counts) == tuple(z["counts"].tolist())
    if it == 0:
        assert np.array_equal(labels, up)


def test_fixtures_cover_the_required_cases():
    seen = {(int(_golden(n)["P"]), int(_golden(n)["num_classes"]), float(_golden(n)["params"][5])) for n in CASES}
    assert {p for p, _, _ in seen} >= {8, 16} and {m for _, m, _ in seen} >= {2, 21}
    assert {it for _, _, it in seen} >= {0.0, 1.0, 5.0}
    assert any(set(np.unique(_golden(n)["segmap"]).tolist()) == {0, 255} for n in CASES)
    assert any(_golden(n)["image"].shape[0] % int(_golden(n)["P"]) for n in CASES)


@pytest.mark.parametrize("name", CASES)
def test_stubbed_reference_command_equals_fixtures(name, tmp_path):
    from oracle import crf_ref, ref_shim
    if not ref_shim.available():
        pytest.skip("reference sources not present")
    from PIL import Image
    ref = ref_shim.load_reference()
    z = _golden(name)
    w1, alpha, beta, w2, gamma, it = z["params"].tolist()
    (tmp_path / f"{name}.jpg").write_bytes(z["jpeg"].tobytes())
    Image.fromarray(z["segmap"]).save(tmp_path / f"{name}.png")
    (tmp_path / "out").mkdir()
    sys.modules["denseCRF"] = crf_ref.make_densecrf_module(unary_eps=float(z["unary_eps"]))
    try:
        ref._extract_crf_segmentations((0, (str(tmp_path / f"{name}.jpg"), str(tmp_path / f"{name}.png"))),
                                       images_root=str(tmp_path), num_classes=int(z["num_classes"]),
                                       output_dir=str(tmp_path / "out"), crf_params=(w1, alpha, beta, w2, gamma, it),
                                       downsample_factor=int(z["P"]))
    finally:
        sys.modules.pop("denseCRF", None)
    assert np.array_equal(np.array(Image.open(tmp_path / "out" / f"{name}.png")), z["labels"])


def test_key_layout_boundary_matches_restatement():
    """dss_crf_segment accepts a batch iff oracle.crf_ref.key_bits puts both lattices' keys in at most 64 bits; at 65
    and more it returns DSS_ERR_UNSUPPORTED before any device work. An accepted layout goes on to the workspace check,
    which a 16-byte workspace fails, so the boundary is probed without a device."""
    from oracle import crf_ref
    _lib = load_pkg("_lib")
    lib = _lib.load()
    import torch
    n0 = lib.dss_kernel_launch_count()
    buf = torch.zeros(1 << 12, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    UNSUP, WS = -4, -3

    def call(shapes, alpha, beta=13.0, gamma=3.0):
        dims = np.array([[H, W, H // 16, W // 16] for H, W in shapes], np.int32)
        return lib.dss_crf_segment(p, p, dims.ctypes.data, len(shapes), 16, 21, 10.0, alpha, beta, 3.0, gamma, 5, 1e-5,
                                   p, None, p, p, 16, None)

    def bits(shapes, alpha, beta=13.0, gamma=3.0):
        H, W = max(h for h, _ in shapes), max(w for _, w in shapes)
        return crf_ref.crf_key_bits(H, W, len(shapes), alpha, beta, gamma)

    voc, big = (375, 500), (500, 500)
    # the worked boundary cases: exactly 64 bits, then one image or one pixel of width more
    assert bits([voc] * 2, 0.05) == (64, 19) and call([voc] * 2, 0.05) == WS
    assert bits([voc] * 3, 0.05)[0] == 65 and call([voc] * 3, 0.05) == UNSUP
    assert bits([voc] * 16, 0.1)[0] == 64 and call([voc] * 16, 0.1) == WS
    assert bits([voc] * 15 + [big], 0.1)[0] == 65 and call([voc] * 15 + [big], 0.1) == UNSUP
    assert bits([voc] * 16, 1.0, beta=0.5)[0] == 66 and call([voc] * 16, 1.0, beta=0.5) == UNSUP
    assert bits([voc] * 16, 80.0) == (43, 22)              # the command's defaults leave 21 bits spare
    # a sweep across the boundary, the spatial lattice's included
    seen = set()
    for shapes in ([voc], [voc] * 2, [voc, big, voc], [big] * 4, [voc] * 16, [voc] * 17, [(48, 64)] * 2):
        for alpha in (0.004, 0.005, 0.008, 0.03, 0.05, 0.07, 0.08, 0.1, 0.13, 1.0):
            for beta, gamma in ((13.0, 3.0), (0.5, 3.0), (13.0, 0.004), (13.0, 1e-3)):
                b = bits(shapes, alpha, beta, gamma)
                top = None if None in b else max(b)                # None: one field alone exceeds 62 bits
                seen.add(top)
                want = WS if top is not None and top <= 64 else UNSUP
                assert call(shapes, alpha, beta, gamma) == want, (shapes, alpha, beta, gamma, b)
    assert {62, 63, 64, 65, 66} <= seen
    assert lib.dss_kernel_launch_count() == n0


def test_crf_entry_points_reject_bad_arguments_before_any_device_work():
    _lib = load_pkg("_lib")
    lib = _lib.load()
    import torch
    n0 = lib.dss_kernel_launch_count()
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    BAD, UNSUP, WS = -1, -4, -3
    dims = np.array([[40, 50, 3, 4], [33, 20, 2, 2]], np.int32)
    dp = dims.ctypes.data
    big = 1 << 40

    def call(images=p, segs=p, dims_=dp, B=2, P=16, M=21, w1=10.0, alpha=80.0, beta=13.0, w2=3.0, gamma=3.0, it=5,
             eps=1e-5, labels=p, info=p, ws=p, ws_bytes=big):
        return lib.dss_crf_segment(images, segs, dims_, B, P, M, w1, alpha, beta, w2, gamma, it, eps, labels, None,
                                   info, ws, ws_bytes, None)

    assert call(images=None) == BAD
    assert call(info=None) == BAD
    assert call(B=0) == BAD
    assert call(P=0) == BAD
    assert call(P=41) == BAD                                   # image 0 is narrower than one patch
    bad_dims = np.array([[40, 50, 0, 4]], np.int32)
    assert call(dims_=bad_dims.ctypes.data, B=1) == BAD
    assert call(M=1) == UNSUP and call(M=65) == UNSUP
    assert call(it=-1) == BAD
    assert call(eps=0.0) == BAD and call(eps=1.5) == BAD
    assert call(alpha=0.0) == BAD and call(gamma=-1.0) == BAD and call(beta=float("inf")) == BAD
    assert call(w1=float("nan")) == BAD
    assert call(ws=p + 8) == BAD
    assert call(ws_bytes=16) == WS
    # keys that do not fit in 64 bits: tiny standard deviations spread the lattice coordinates
    assert call(alpha=1e-3, beta=1e-3) == UNSUP
    assert b"64 bits" in lib.dss_last_error()
    assert lib.dss_crf_workspace_bytes(dp, 2, 1) == 0 and lib.dss_crf_workspace_bytes(dp, 2, 65) == 0
    assert lib.dss_crf_workspace_bytes(bad_dims.ctypes.data, 1, 21) == 0
    assert lib.dss_crf_workspace_bytes(dp, 2, 21) > 0
    # lattice filter
    assert lib.dss_op_lattice_filter(None, 10, 5, p, 4, 0, p, None, p, big, None) == BAD
    assert lib.dss_op_lattice_filter(p, 0, 5, p, 4, 0, p, None, p, big, None) == BAD
    assert lib.dss_op_lattice_filter(p, 10, 3, p, 4, 0, p, None, p, big, None) == UNSUP
    assert lib.dss_op_lattice_filter(p, 10, 5, p, 65, 0, p, None, p, big, None) == UNSUP
    assert lib.dss_op_lattice_filter(p, 10, 5, p, 4, 0, p, None, p + 8, big, None) == BAD
    assert lib.dss_op_lattice_filter(p, 10, 5, p, 4, 0, p, None, p, 16, None) == WS
    assert lib.dss_lattice_filter_workspace_bytes(10, 3, 4) == 0 and lib.dss_lattice_filter_workspace_bytes(10, 2, 4) > 0
    assert lib.dss_kernel_launch_count() == n0
