"""Dense CRF on the GPU (csrc/crf.cu) against the float64 restatement in oracle/crf_ref.py, at VOC size and at the
kernel's edges: the lattice filter on VOC-size and degenerate point sets within a derived fp32 error bound, the mean
field at every class-lane width, label-map and image shapes, closed forms, batches of identical images, a production
batch, key layouts up to exactly 64 bits, and the buffers each entry point may touch."""
import numpy as np
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

Q_TOL = 1e-5          # DESIGN §5: Q within 1e-5 of the float64 lattice mean field
CLEAR = 1e-4          # labels are compared where the oracle's top-two gap exceeds this (as in tests/test_crf_gpu.py)
DEFAULTS = dict(w1=10.0, alpha=80.0, beta=13.0, w2=3.0, gamma=3.0)
# G = next_pow2(ceil(M / 4)) lanes per pixel: 1 (M <= 4), 2, 4 (M 9 .. 16), 8, 16 (M 33 .. 64); multiples of 4 have no
# padded class
LANE_M = [2, 3, 4, 5, 8, 9, 12, 16, 17, 21, 32, 33, 48, 64]
VOC_H, VOC_W = 375, 500


def _blobs(H, W, seed):
    return load_pkg("synth").blobs_image(H, W, seed).numpy()


def _run(cuda, images, segs, M, P, **kw):
    """dense_crf -> (labels, Q [HW, M], info) per image, as numpy."""
    crf = load_pkg("crf")
    labels, Q, info = crf.dense_crf(images, segs, M, P, return_prob=True, device=cuda, **kw)
    info = info.cpu().numpy()
    return [(l.cpu().numpy(), q.reshape(-1, M).cpu().numpy(), tuple(info[b].tolist()))
            for b, (l, q) in enumerate(zip(labels, Q))]


def _oracle(image, seg, M, P, params, eps):
    from oracle import crf_ref
    H, W = image.shape[:2]
    return crf_ref.mean_field(image, np.eye(M)[crf_ref.upsample_labels(seg, H, W, P)], params, eps)


def _params(kw, it):
    return (kw["w1"], kw["alpha"], kw["beta"], kw["w2"], kw["gamma"], it)


def _check_against_oracle(got, Q_ref, counts, what=""):
    """Q within Q_TOL, lattice point counts equal, labels (first-wins argmax) equal wherever the oracle's top-two gap
    is clear."""
    labels, q, info = got
    err = float(np.abs(q - Q_ref).max())
    assert err <= Q_TOL, (what, err)
    assert info == tuple(counts), (what, info, counts)
    want = Q_ref.argmax(1)
    top2 = np.sort(Q_ref, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > CLEAR
    assert np.array_equal(labels.ravel()[clear], want[clear]), what


def _same_bits(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32)) and a[2] == b[2]


# ---------------------------------------------------------------------------------------------------- lattice filter
def _voc_image(name):
    if name == "blobs":
        return _blobs(VOC_H, VOC_W, 0)
    img = np.full((VOC_H, VOC_W, 3), 120, np.uint8)
    if name == "two_tone":
        img[:, VOC_W // 2:] = (20, 200, 90)
    return img


def _voc_features(name, d):
    from oracle import crf_ref
    if name == "noise":
        return (np.random.default_rng(d).normal(size=(VOC_H * VOC_W, d)) * 2.5).astype(np.float32)
    fb, fs = crf_ref.crf_features(_voc_image(name), DEFAULTS["alpha"], DEFAULTS["beta"], DEFAULTS["gamma"])
    return (fb if d == 5 else fs).astype(np.float32)


@pytest.fixture(scope="module")
def voc_lattice():
    """float64 lattices of the VOC-size point sets, built once per module (2 - 3 s each on the CPU)."""
    from oracle import crf_ref
    cache = {}

    def get(name, d):
        if (name, d) not in cache:
            f = _voc_features(name, d)
            cache[(name, d)] = (f, crf_ref.Lattice(f.astype(np.float64)))
        return cache[(name, d)]
    return get


def _filter_and_bound(cuda, f, lat, C, normalize, seed):
    crf = load_pkg("crf")
    v = np.random.default_rng(seed).random((f.shape[0], C)).astype(np.float32)
    out, points = crf.lattice_filter(torch.from_numpy(f).to(cuda), torch.from_numpy(v).to(cuda), normalize)
    want = lat.filter(v.astype(np.float64), normalize)
    err = np.abs(out.cpu().numpy().astype(np.float64) - want)
    return points, err, lat.fp32_error_bound(v, normalize), np.abs(want).max()


# The three images are the issue's extremes at the default parameters: a constant colour puts 16 500 contributions into
# its busiest bilateral lattice point, blobs 9 400, i.i.d. noise features leave almost every point with one or two.
# The spatial lattice of all three images is the same, so it is run once.
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("name,d", [("constant", 5), ("two_tone", 5), ("blobs", 5), ("blobs", 2), ("noise", 5),
                                    ("noise", 2)])
def test_lattice_filter_at_voc_size_within_fp32_bound(cuda, voc_lattice, name, d, normalize):
    f, lat = voc_lattice(name, d)
    points, err, bound, scale = _filter_and_bound(cuda, f, lat, 5, normalize, seed=d)
    assert points == lat.points
    # componentwise: Lattice.fp32_error_bound derives it from every lattice point's contribution count (see there)
    worst = float((err / bound).max())
    assert (err <= bound).all(), (worst, lat.contributions().max())
    # the 1e-5 of the output's max that the small point sets are held to (tests/test_crf_gpu.py) holds here too: the
    # constant colour, normalised, measures the most
    assert err.max() <= 1e-5 * scale, (err.max() / scale, lat.contributions().max())


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("d", [2, 5])
@pytest.mark.parametrize("kind", ["identical", "offset", "negative"])
def test_lattice_filter_on_degenerate_point_sets(cuda, kind, d, normalize):
    from oracle import crf_ref
    rng = np.random.default_rng(7 * d + len(kind))
    N = 257
    if kind == "identical":
        f = np.tile(rng.normal(size=(1, d)) * 3.0, (N, 1))
    elif kind == "offset":        # far from the origin: keys offset by about 1e5 in every coordinate
        f = rng.normal(size=(N, d)) * 2.5 + 1e5
    else:
        f = -np.abs(rng.normal(size=(N, d))) * 4.0 - 50.0
    f = f.astype(np.float32)
    lat = crf_ref.Lattice(f.astype(np.float64))
    if kind == "identical":
        assert lat.points == d + 1
    points, err, bound, scale = _filter_and_bound(cuda, f, lat, 17, normalize, seed=d)
    assert points == lat.points
    assert (err <= bound).all(), float((err / bound).max())
    assert err.max() <= 1e-5 * scale


# ---------------------------------------------------------------------------------------------------- mean field
@pytest.mark.parametrize("M", LANE_M)
def test_mean_field_at_every_lane_width(cuda, M):
    P, H, W = 8, 48, 64
    img = _blobs(H, W, 200 + M)
    seg = np.random.default_rng(M).integers(0, M, (H // P, W // P)).astype(np.uint8)
    kw = dict(DEFAULTS, unary_eps=0.2)
    Qs, _, counts = _oracle(img, seg, M, P, _params(kw, 5), 0.2)
    for it in (0, 1, 5):
        got = _run(cuda, [img], [seg], M, P, it=it, **kw)[0]
        _check_against_oracle(got, Qs[it], counts, (M, it))
        if it == 5:
            assert (got[0].ravel() != Qs[0].argmax(1)).any()    # eps = 0.2 lets labels move


@pytest.mark.parametrize("M", LANE_M)
def test_closed_forms_at_every_lane_width(cuda, M):
    from oracle import crf_ref
    P, H, W = 8, 48, 64
    img = _blobs(H, W, 300 + M)
    seg = np.random.default_rng(100 + M).integers(0, M, (H // P, W // P)).astype(np.uint8)
    up = crf_ref.upsample_labels(seg, H, W, P).ravel()
    # no pairwise terms: Q = softmax(-U) at every iteration, 1 / (1 + (M - 1) eps) at the label and eps times that
    # elsewhere. The kernel rounds log(eps) to fp32 (|log eps| u relative in exp), expf (2 ulp = 4 u), sums M terms
    # (M - 1 roundings) and divides (u).
    eps = 0.2
    labels, q, _ = _run(cuda, [img], [seg], M, P, it=3, **dict(DEFAULTS, w1=0.0, w2=0.0), unary_eps=eps)[0]
    z = 1.0 / (1.0 + (M - 1) * eps)
    want = np.where(np.arange(M)[None, :] == up[:, None], z, eps * z)
    rel = (M + 5 + abs(np.log(eps))) * crf_ref.U32
    assert (np.abs(q - want) <= rel * want).all(), float((np.abs(q - want) / want).max())
    off = np.where(np.arange(M)[None, :] == up[:, None], np.nan, q)
    assert (np.nanmax(off, 1) == np.nanmin(off, 1)).all()      # every class off the label carries the same bits
    assert np.array_equal(labels.ravel(), up)
    # no unary (eps = 1): every class of every pixel holds the same logits, so Q = fl(1 / M) bit for bit and the argmax
    # tie goes to class 0 across all lanes
    labels, q, _ = _run(cuda, [img], [seg], M, P, it=2, **DEFAULTS, unary_eps=1.0)[0]
    assert (q == np.float32(1.0 / M)).all()
    assert not labels.any()


@pytest.mark.parametrize("P", [8, 14, 16])
def test_shapes_and_label_maps(cuda, P):
    """Images of one patch, one patch row, tall and thin, not multiples of P, and label maps of other sizes than
    H // P x W // P (the command takes any PNG size): one ragged call per iteration count."""
    from oracle import crf_ref
    cases = [(P, P, 1, 1), (P + 3, 6 * P + 5, 1, 6), (9 * P + 2, P, 9, 1), (3 * P + 5, 4 * P + 7, 3, 4),
             (3 * P + 5, 4 * P + 7, 4, 4), (2 * P, 3 * P, 5, 2), (2 * P + 1, 2 * P + 1, 7, 3)]
    M = 5
    rng = np.random.default_rng(P)
    imgs = [_blobs(H, W, 500 + i) for i, (H, W, _, _) in enumerate(cases)]
    segs = [rng.integers(0, M, (sh, sw)).astype(np.uint8) for _, _, sh, sw in cases]
    kw = dict(DEFAULTS, unary_eps=0.2)
    for (H, W, _, _), img, seg, got in zip(cases, imgs, segs, _run(cuda, imgs, segs, M, P, it=0, **kw)):
        assert np.array_equal(got[0], crf_ref.upsample_labels(seg, H, W, P)), (H, W, seg.shape)
    for (H, W, _, _), img, seg, got in zip(cases, imgs, segs, _run(cuda, imgs, segs, M, P, it=2, **kw)):
        Qs, _, counts = _oracle(img, seg, M, P, _params(kw, 2), 0.2)
        _check_against_oracle(got, Qs[2], counts, (H, W, seg.shape))


# ---------------------------------------------------------------------------------------------------- batches, layouts
@pytest.mark.parametrize("k", [2, 3, 16, 17])
def test_identical_copies_are_kept_apart_by_the_image_bits(cuda, k):
    """Copies share every lattice coordinate: only the image index in the key keeps their lattices apart."""
    P, M = 16, 21
    img = _blobs(96, 128, 11)
    seg = np.random.default_rng(11).integers(0, M, (6, 8)).astype(np.uint8)
    kw = dict(DEFAULTS, unary_eps=0.2, it=3)
    solo = _run(cuda, [img], [seg], M, P, **kw)[0]
    for b, row in enumerate(_run(cuda, [img] * k, [seg] * k, M, P, **kw)):
        assert _same_bits(row, solo), b


def _voc_label_map(H, W, P, M, seed):
    """The label maps of tools/crf_probe.py: six random rectangles of labels 1 .. M - 1 on background 0."""
    rng = np.random.default_rng(seed)
    m = np.zeros((H // P, W // P), np.uint8)
    for _ in range(6):
        y, x = rng.integers(0, m.shape[0]), rng.integers(0, m.shape[1])
        m[y:y + rng.integers(2, 10), x:x + rng.integers(2, 12)] = rng.integers(1, M)
    return m


@pytest.fixture(scope="module")
def production(cuda):
    """16 VOC-shaped images, 21 classes, the command's defaults: the batch, every image alone, and the float64 oracle
    of three rows (the largest shape among them)."""
    P, M = 16, 21
    kw = dict(DEFAULTS, unary_eps=1e-5, it=5)
    shapes = load_pkg("synth").voc_shapes(16, seed=0)
    imgs = [_blobs(H, W, i) for i, (H, W) in enumerate(shapes)]
    segs = [_voc_label_map(H, W, P, M, i) for i, (H, W) in enumerate(shapes)]
    batch = _run(cuda, imgs, segs, M, P, **kw)
    solo = [_run(cuda, [im], [s], M, P, **kw)[0] for im, s in zip(imgs, segs)]
    largest = max(range(16), key=lambda b: shapes[b][0] * shapes[b][1])
    rows = sorted({largest, 0, 1})
    oracle = {b: _oracle(imgs[b], segs[b], M, P, _params(kw, 5), 1e-5) for b in rows}
    return dict(P=P, M=M, kw=kw, shapes=shapes, imgs=imgs, segs=segs, batch=batch, solo=solo, largest=largest,
                oracle=oracle)


def test_production_batch_rows_equal_solo_runs_and_float64(production):
    pr = production
    for b in range(16):
        assert _same_bits(pr["batch"][b], pr["solo"][b]), (b, pr["shapes"][b])
    assert pr["largest"] in pr["oracle"] and pr["shapes"][pr["largest"]] == (500, 500)
    for b, (Qs, _, counts) in pr["oracle"].items():
        _check_against_oracle(pr["batch"][b], Qs[-1], counts, pr["shapes"][b])


def test_mean_field_at_voc_size_on_two_flat_colours(cuda):
    """The busiest lattice points there are: each flat half splats some 16 500 pixels into one bilateral point."""
    P, M = 16, 21
    img = _voc_image("two_tone")
    seg = _voc_label_map(VOC_H, VOC_W, P, M, 7)
    kw = dict(DEFAULTS, unary_eps=1e-5, it=5)
    Qs, _, counts = _oracle(img, seg, M, P, _params(kw, 5), 1e-5)
    _check_against_oracle(_run(cuda, [img], [seg], M, P, **kw)[0], Qs[-1], counts, "two flat colours")


def test_layout_invariance_next_to_a_500x500_companion(cuda, production):
    """Field widths follow the batch's largest image; the lattice, its point order and its summation order do not."""
    pr = production
    b = 0                                                   # a 500 x 375 image
    comp = _blobs(500, 500, 99)
    comp_seg = _voc_label_map(500, 500, pr["P"], pr["M"], 99)
    rows = _run(cuda, [comp, pr["imgs"][b]], [comp_seg, pr["segs"][b]], pr["M"], pr["P"], **pr["kw"])
    assert _same_bits(rows[1], pr["solo"][b])


def test_key_layouts_of_63_and_64_bits(cuda):
    """48 x 64 images at alpha = 0.008 need 63 bilateral key bits alone and 64 next to a second image, whose index then
    sits in bit 63; alpha = 0.005 fills all 64 bits with coordinates. A third image would need 65 bits: rejected."""
    from oracle import crf_ref
    _lib = load_pkg("_lib")
    P, M, H, W = 8, 5, 48, 64
    img, other = _blobs(H, W, 21), _blobs(H, W, 22)
    rng = np.random.default_rng(21)
    seg, oseg = (rng.integers(0, M, (H // P, W // P)).astype(np.uint8) for _ in range(2))
    for alpha, B, bits in ((0.008, 1, 63), (0.008, 2, 64), (0.008, 3, 65), (0.005, 1, 64)):
        assert crf_ref.crf_key_bits(H, W, B, alpha, DEFAULTS["beta"], DEFAULTS["gamma"])[0] == bits
    kw = dict(DEFAULTS, alpha=0.008, unary_eps=0.2, it=3)
    alone = _run(cuda, [img], [seg], M, P, **kw)[0]
    pair = _run(cuda, [other, img], [oseg, seg], M, P, **kw)
    assert _same_bits(pair[1], alone)
    Qs, _, counts = _oracle(img, seg, M, P, _params(kw, 3), 0.2)
    _check_against_oracle(pair[1], Qs[-1], counts, "64 bits, image bit 63")
    Qs, _, counts = _oracle(other, oseg, M, P, _params(kw, 3), 0.2)
    _check_against_oracle(pair[0], Qs[-1], counts, "64 bits, image 0")
    with pytest.raises(_lib.DssError, match="64 bits"):
        _run(cuda, [other, other, img], [oseg, oseg, seg], M, P, **kw)
    kw = dict(kw, alpha=0.005)
    Qs, _, counts = _oracle(img, seg, M, P, _params(kw, 3), 0.2)
    _check_against_oracle(_run(cuda, [img], [seg], M, P, **kw)[0], Qs[-1], counts, "64 coordinate bits")


# ---------------------------------------------------------------------------------------------------- buffers
TAIL = 4096   # bytes of canary after every buffer


def _padded(n_bytes, fill, cuda):
    return torch.full((n_bytes + TAIL,), fill, dtype=torch.uint8, device=cuda)


def test_crf_segment_stays_inside_its_buffers_and_reads_no_stale_workspace(cuda):
    """A workspace of exactly the reported size and outputs of exactly their size, each followed by a canary, once
    filled with zeros and once with 0xFF (NaN as fp32): no canary changes, and the outputs are the same bits."""
    _lib = load_pkg("_lib")
    lib = _lib.load()
    P, M = 8, 7
    shapes = [(40, 56, 5, 7), (33, 70, 4, 8), (64, 48, 8, 6)]
    rng = np.random.default_rng(5)
    imgs = [_blobs(H, W, 600 + i) for i, (H, W, _, _) in enumerate(shapes)]
    segs = [rng.integers(0, M, (sh, sw)).astype(np.uint8) for _, _, sh, sw in shapes]
    dims = np.array(shapes, np.int32)
    B, N = len(shapes), sum(H * W for H, W, _, _ in shapes)
    need = int(lib.dss_crf_workspace_bytes(dims.ctypes.data, B, M))
    assert need > 0
    img_d = torch.from_numpy(np.concatenate([i.ravel() for i in imgs])).to(cuda)
    seg_d = torch.from_numpy(np.concatenate([s.ravel() for s in segs])).to(cuda)
    runs = []
    for fill in (0x00, 0xFF):
        ws, lab, prob, info = (_padded(n, fill, cuda) for n in (need, N, 4 * N * M, 4 * 2 * B))
        assert ws.data_ptr() % 256 == 0
        _lib.check(lib.dss_crf_segment(img_d.data_ptr(), seg_d.data_ptr(), dims.ctypes.data, B, P, M, 10.0, 80.0, 13.0,
                                       3.0, 3.0, 2, 0.2, lab.data_ptr(), prob.data_ptr(), info.data_ptr(), ws.data_ptr(),
                                       need, _lib.stream_ptr(cuda)), "dss_crf_segment")
        torch.cuda.synchronize()
        for t, n in ((ws, need), (lab, N), (prob, 4 * N * M), (info, 8 * B)):
            assert bool((t[n:] == fill).all()), (fill, n)
        runs.append([t[:n].cpu() for t, n in ((lab, N), (prob, 4 * N * M), (info, 8 * B))])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    assert torch.equal(img_d.cpu(), torch.from_numpy(np.concatenate([i.ravel() for i in imgs])))


@pytest.mark.parametrize("d", [2, 5])
@pytest.mark.parametrize("normalize", [0, 1])
def test_lattice_filter_stays_inside_its_buffers_and_reads_no_stale_workspace(cuda, d, normalize):
    _lib = load_pkg("_lib")
    lib = _lib.load()
    N, C = 1001, 5
    rng = np.random.default_rng(d)
    f = torch.from_numpy((rng.normal(size=(N, d)) * 2.5).astype(np.float32)).to(cuda)
    v = torch.from_numpy(rng.random((N, C)).astype(np.float32)).to(cuda)
    need = int(lib.dss_lattice_filter_workspace_bytes(N, d, C))
    assert need > 0
    runs = []
    for fill in (0x00, 0xFF):
        ws, out, pts = (_padded(n, fill, cuda) for n in (need, 4 * N * C, 4))
        _lib.check(lib.dss_op_lattice_filter(f.data_ptr(), N, d, v.data_ptr(), C, normalize, out.data_ptr(),
                                             pts.data_ptr(), ws.data_ptr(), need, _lib.stream_ptr(cuda)),
                   "dss_op_lattice_filter")
        torch.cuda.synchronize()
        for t, n in ((ws, need), (out, 4 * N * C), (pts, 4)):
            assert bool((t[n:] == fill).all()), (fill, n)
        runs.append([out[:4 * N * C].cpu(), pts[:4].cpu()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
