"""Dense CRF on the GPU (csrc/crf.cu): the lattice filter against the float64 restatement, the mean field against the
reference's stored outputs (tests/golden/ref_crf_*.npz) and against the exact-filter oracle, determinism across batches
and runs, the 64-bit key limit, and the extract_crf_segmentations command end to end."""
import numpy as np
import pytest
import torch

from conftest import ROOT, load_pkg

pytestmark = pytest.mark.gpu

GOLDEN = ROOT / "tests" / "golden"
CASES = sorted(p.stem[len("ref_crf_"):] for p in GOLDEN.glob("ref_crf_*.npz"))
LABEL_AGREEMENT = 0.95   # lattice vs exact mean-field labels, measured on the CPU (tests/test_cpu_crf.py)


def _golden(name):
    return np.load(GOLDEN / f"ref_crf_{name}.npz", allow_pickle=False)


def _case(name):
    z = _golden(name)
    w1, alpha, beta, w2, gamma, it = z["params"].tolist()
    image = z["image"]
    H, W = image.shape[:2]
    P, M = int(z["P"]), int(z["num_classes"])
    seg = load_pkg("crf").prepare_segmap(z["segmap"], H, W, P, M)
    kw = dict(w1=w1, alpha=alpha, beta=beta, w2=w2, gamma=gamma, it=int(it), unary_eps=float(z["unary_eps"]))
    return z, image, seg, P, M, kw


# "random" / "image": 1001 random points and a 37 x 45 image with 7 channels; "n<N>_c<C>": N random points with C
# channels (every channel tail of the float4 class rows, up to 64; N around one 256-thread block); "image_c<C>"
SOURCES = ["random", "image", "n1_c1", "n2_c3", "n7_c4", "n255_c5", "n256_c8", "n257_c16", "n1001_c17", "n1001_c33",
           "image_c64"]


@pytest.mark.parametrize("d", [2, 5])
@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("normalize", [False, True])
def test_lattice_filter_matches_float64_restatement(cuda, d, source, normalize):
    from oracle import crf_ref
    crf = load_pkg("crf")
    rng = np.random.default_rng(d * 10 + (source == "image") if source in ("random", "image")
                                else (d, SOURCES.index(source)))
    kind, N, C = source, 1001, 7
    if "_" in source:
        kind, c = source.split("_")
        C = int(c[1:])
        if kind != "image":
            kind, N = "random", int(kind[1:])
    if kind == "random":
        f = (rng.normal(size=(N, d)) * 2.5).astype(np.float32)
    else:
        img = load_pkg("synth").blobs_image(37, 45, 7).numpy()
        fb, fs = crf_ref.crf_features(img, 80, 13, 3)
        f = (fb if d == 5 else fs).astype(np.float32)
    v = rng.random((f.shape[0], C)).astype(np.float32)
    out, points = crf.lattice_filter(torch.from_numpy(f).to(cuda), torch.from_numpy(v).to(cuda), normalize)
    lat = crf_ref.Lattice(f.astype(np.float64))
    want = lat.filter(v.astype(np.float64), normalize)
    assert points == lat.points
    err = np.abs(out.cpu().numpy() - want).max()
    assert err <= 1e-5 * np.abs(want).max(), err


@pytest.mark.parametrize("name", CASES)
def test_dense_crf_matches_reference_fixtures(cuda, name):
    from oracle import crf_ref
    crf = load_pkg("crf")
    z, image, seg, P, M, kw = _case(name)
    labels, Q, info = crf.dense_crf([image], [seg], M, P, return_prob=True, device=cuda, **kw)
    q = Q[0].reshape(-1, M).cpu().numpy().astype(np.float64)
    assert np.abs(q - z["Q"]).max() <= 1e-5
    assert tuple(info[0].cpu().tolist()) == tuple(z["counts"].tolist())
    got, want = labels[0].cpu().numpy(), z["labels"]
    top2 = np.sort(z["Q"], 1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0] > 1e-4).reshape(want.shape)
    assert np.array_equal(got[clear], want[clear])
    assert (~clear).mean() < 1e-3
    if kw["it"] == 0:
        assert np.array_equal(got, crf_ref.upsample_labels(seg, *image.shape[:2], P))


def test_dense_crf_label_agreement_with_exact_filter(cuda):
    from oracle import crf_ref
    crf = load_pkg("crf")
    synth = load_pkg("synth")
    worst = 1.0
    for seed in range(3):
        img = synth.blobs_image(64, 64, 100 + seed).numpy()
        seg = np.random.default_rng(seed).integers(0, 4, (8, 8)).astype(np.uint8)
        prob = np.eye(4)[crf_ref.upsample_labels(seg, 64, 64, 8)]
        _, l_ex, _ = crf_ref.mean_field(img, prob, (10, 80, 13, 3, 3, 5), 0.2, filter="exact")
        labels, _, _ = crf.dense_crf([img], [seg], 4, 8, it=5, unary_eps=0.2, device=cuda)
        worst = min(worst, float((labels[0].cpu().numpy() == l_ex).mean()))
    assert worst >= LABEL_AGREEMENT, worst


def test_dense_crf_is_bitwise_deterministic_across_batches_and_runs(cuda):
    crf = load_pkg("crf")
    synth = load_pkg("synth")
    _, image, seg, P, M, kw = _case("p16_c21_it5")
    rng = np.random.default_rng(3)
    others = []
    for i, (H, W) in enumerate([(97, 130), (33, 200), (160, 48)]):
        others.append((synth.blobs_image(H, W, 40 + i).numpy(), rng.integers(0, M, (H // P, W // P)).astype(np.uint8)))
    alone = crf.dense_crf([image], [seg], M, P, return_prob=True, device=cuda, **kw)
    again = crf.dense_crf([image], [seg], M, P, return_prob=True, device=cuda, **kw)
    mixed = crf.dense_crf([others[0][0], image, others[1][0], others[2][0]], [others[0][1], seg, others[1][1], others[2][1]],
                          M, P, return_prob=True, device=cuda, **kw)
    for run, k in ((again, 0), (mixed, 1)):
        assert torch.equal(alone[0][0], run[0][k])
        assert torch.equal(alone[1][0].view(torch.int32), run[1][k].view(torch.int32))
        assert torch.equal(alone[2][0], run[2][k])
    for j, k in ((0, 0), (1, 2), (2, 3)):   # the other images alone equal their batch rows as well
        solo = crf.dense_crf([others[j][0]], [others[j][1]], M, P, return_prob=True, device=cuda, **kw)
        assert torch.equal(solo[0][0], mixed[0][k])
        assert torch.equal(solo[1][0].view(torch.int32), mixed[1][k].view(torch.int32))


def test_keys_beyond_64_bits_are_rejected(cuda):
    _lib = load_pkg("_lib")
    crf = load_pkg("crf")
    _, image, seg, P, M, kw = _case("p16_c21_it5")
    kw.update(alpha=1e-3, beta=1e-3)
    with pytest.raises(_lib.DssError, match="64 bits"):
        crf.dense_crf([image], [seg], M, P, device=cuda, **kw)


def test_extract_crf_segmentations_command(cuda, tmp_path, capsys):
    from PIL import Image
    ex = load_pkg("extract")
    for name in CASES:
        z, image, seg, P, M, kw = _case(name)
        root = tmp_path / name
        idir, sdir, odir = root / "images", root / "segs", root / "out"
        idir.mkdir(parents=True)
        sdir.mkdir()
        (idir / f"{name}.jpg").write_bytes(z["jpeg"].tobytes())
        Image.fromarray(z["segmap"]).save(sdir / f"{name}.png")
        args = dict(num_classes=M, downsample_factor=P, w1=kw["w1"], alpha=kw["alpha"], beta=kw["beta"], w2=kw["w2"],
                    gamma=kw["gamma"], it=float(kw["it"]), unary_eps=kw["unary_eps"], yes=True)
        ex.extract_crf_segmentations(str(idir), str(idir), str(sdir), str(odir), **args)
        out = Image.open(odir / f"{name}.png")
        assert out.mode == "L" and out.size == (image.shape[1], image.shape[0])
        got, want = np.array(out), z["labels"]
        top2 = np.sort(z["Q"], 1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0] > 1e-4).reshape(want.shape)
        assert np.array_equal(got[clear], want[clear]), name
        mtime = (odir / f"{name}.png").stat().st_mtime_ns
        capsys.readouterr()
        ex.extract_crf_segmentations(str(idir), str(idir), str(sdir), str(odir), **args)
        assert "Skipping existing file" in capsys.readouterr().out
        assert (odir / f"{name}.png").stat().st_mtime_ns == mtime


def test_command_rejects_labels_beyond_num_classes(cuda, tmp_path):
    from PIL import Image
    ex = load_pkg("extract")
    z = _golden("p16_c21_it5")
    (tmp_path / "i").mkdir()
    (tmp_path / "s").mkdir()
    (tmp_path / "i" / "a.jpg").write_bytes(z["jpeg"].tobytes())
    seg = z["segmap"].copy()
    seg[0, 0] = 30
    Image.fromarray(seg).save(tmp_path / "s" / "a.png")
    with pytest.raises(ValueError, match="a.png: label 30"):
        ex.extract_crf_segmentations(str(tmp_path / "i"), str(tmp_path / "i"), str(tmp_path / "s"), str(tmp_path / "o"),
                                     yes=True)
