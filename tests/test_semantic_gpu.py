"""-m gpu: the semantic-segmentation stages (csrc/cluster.cu) -- segment boxes against the scipy oracle and the
reference's stored outputs, covariance / PCA against float64 numpy and scikit-learn, data-set K-means (planted
partitions, inertia against scikit-learn, bit reproducibility), and the whole chain from images to pseudo-label maps."""
import ast

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import ROOT, load_pkg

pytestmark = pytest.mark.gpu
GOLDEN = ROOT / "tests" / "golden"


def _rows(d):
    return np.array([[s, *b, *o] for s, b, o in zip(d["segment_indices"], d["bboxes"], d["bboxes_original_resolution"])],
                    np.int64).reshape(-1, 9)


def _random_label_map(rng, H, W, n_labels):
    m = np.zeros((H, W), np.uint8)
    labels = rng.choice(np.arange(1, 256), size=n_labels, replace=False)
    for v in labels:
        y, x = rng.integers(0, H), rng.integers(0, W)
        h, w = rng.integers(1, max(2, H // 2)), rng.integers(1, max(2, W // 2))
        m[y:y + h, x:x + w] = v
    return m


@pytest.mark.parametrize("H,W", [(7, 11), (14, 14), (30, 30), (23, 41), (60, 60), (80, 80)])
def test_segment_boxes_equal_the_oracle(cuda, H, W):
    from oracle import bbox_ref
    cluster = load_pkg("cluster"); ex = load_pkg("extract")
    rng = np.random.default_rng(H * 1000 + W)
    maps = np.stack([_random_label_map(rng, H, W, int(rng.integers(1, 41))) for _ in range(6)])
    for ne, nd in [(0, 0), (2, 3), (5, 1), (1, 5), (3, 3)]:
        boxes, present = cluster.segment_bboxes(torch.from_numpy(maps).to(cuda), ne, nd)
        boxes, present = boxes.cpu().numpy(), present.cpu().numpy()
        for b in range(len(maps)):
            assert np.array_equal(np.flatnonzero(present[b]), np.unique(maps[b]))
            for skip in (True, False):
                want = bbox_ref.extract_bbox(maps[b], "x", 16, ne, nd, skip)
                got = ex._bbox_dict("x", 16, boxes[b], present[b], skip)
                assert np.array_equal(_rows(got), _rows(want)), (H, W, ne, nd, skip, b)


def test_extract_bboxes_matches_reference_fixtures(cuda, tmp_path):
    ex = load_pkg("extract")
    z = np.load(GOLDEN / "ref_bboxes.npz")
    cases = ast.literal_eval(str(z["cases"]))
    fdir, sdir = tmp_path / "f", tmp_path / "s"
    fdir.mkdir(); sdir.mkdir()
    names = sorted(k[4:] for k in z.files if k.startswith("map_"))
    for name in names:
        m = z[f"map_{name}"]
        torch.save({"id": name, "patch_size": 16, "shape": (1, 3, m.shape[0] * 16 + 5, m.shape[1] * 16), "k": torch.zeros(1)},
                   fdir / f"{name}.pth")
        Image.fromarray(m).save(sdir / f"{name}.png")
    for ci, (ne, nd, skip, ds) in enumerate(cases):
        out_file = tmp_path / "out" / f"bboxes{ci}.pth"
        ex.extract_bboxes(str(fdir), str(sdir), str(out_file), num_erode=ne, num_dilate=nd, skip_bg_index=skip,
                          downsample_factor=ds)
        out = torch.load(out_file, weights_only=False)
        assert [d["id"] for d in out] == names
        for d in out:
            assert np.array_equal(_rows(d), z[f"case{ci}_{d['id']}"]), (ci, d["id"])
            assert d["format"] == "(xmin, ymin, xmax, ymax)"
            assert type(d["segment_indices"][0]) is int and type(d["bboxes"][0][0]) is np.int64


def test_covariance_matches_float64(cuda):
    cluster = load_pkg("cluster")
    g = torch.Generator().manual_seed(0)
    X = (torch.randn(20000, 384, generator=g) * torch.linspace(0.1, 2.0, 384) + 0.3).float()
    mean, cov = cluster.covariance(X.to(cuda))
    x64 = X.double().numpy()
    want = np.cov(x64, rowvar=False)
    got = cov[:, :384].double().cpu().numpy()
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    assert np.abs(mean.double().cpu().numpy() - x64.mean(0)).max() <= 1e-6 * np.abs(x64.mean(0)).max()
    assert torch.equal(cov[:, 384:].cpu(), torch.zeros(384, cov.shape[1] - 384))


def test_pca_subspace_matches_sklearn(cuda):
    from scipy.linalg import subspace_angles
    from sklearn.decomposition import PCA
    cluster = load_pkg("cluster")
    g = np.random.default_rng(1)
    M, d, p = 30000, 384, 32
    basis = np.linalg.qr(g.normal(size=(d, d)))[0]
    scales = np.concatenate([np.linspace(5.0, 2.0, p), np.full(d - p, 0.2)])    # clear gap after pca_dim
    X = ((g.normal(size=(M, d)) * scales) @ basis.T + 0.5).astype(np.float32)
    mean, cov = cluster.covariance(torch.from_numpy(X).to(cuda))
    V = cluster.pca_components(cov, d, p).cpu().numpy()
    sk = PCA(p).fit(X)
    assert np.max(subspace_angles(V.T.astype(np.float64), sk.components_.T.astype(np.float64))) <= 1e-4
    Y = cluster.pca(torch.from_numpy(X).to(cuda), p).cpu().numpy()
    Ysk = sk.transform(X)
    signs = np.sign((Y * Ysk).sum(0))
    assert np.abs(Y * signs - Ysk).max() <= 1e-3 * np.abs(Ysk).max()


def _planted(seed, M, dims, k, spread, noise):
    g = np.random.default_rng(seed)
    centres = g.normal(size=(k, dims)) * spread
    truth = g.integers(0, k, size=M)
    X = (centres[truth] + noise * g.normal(size=(M, dims))).astype(np.float32)
    return X, truth


def _same_partition(a, b):
    pairs = set(zip(a.tolist(), b.tolist()))
    return len(pairs) == len(set(a.tolist())) == len(set(b.tolist()))


def test_kmeans_recovers_a_planted_partition(cuda):
    cluster = load_pkg("cluster")
    X, truth = _planted(0, 100000, 32, 21, 3.0, 0.1)
    Xd = torch.from_numpy(X).to(cuda)
    for seed in range(5):
        labels, centres, info, _ = cluster.kmeans(Xd, 21, seed=seed)
        lab = labels.cpu().numpy()
        assert lab.dtype == np.int32 and lab.min() >= 0 and lab.max() < 21
        assert int(info[1]) == 1
        assert _same_partition(lab, truth), seed


def _inertia(X, labels):
    X = X.astype(np.float64)
    s = 0.0
    for c in np.unique(labels):
        pts = X[labels == c]
        s += ((pts - pts.mean(0)) ** 2).sum()
    return s


def test_kmeans_inertia_is_on_par_with_sklearn(cuda):
    from sklearn.cluster import KMeans, MiniBatchKMeans
    cluster = load_pkg("cluster")
    X, _ = _planted(3, 20000, 16, 12, 1.0, 0.7)      # overlapping mixture
    Xd = torch.from_numpy(X).to(cuda)
    ours, mb, full = [], [], []
    for seed in range(5):
        ours.append(_inertia(X, cluster.kmeans(Xd, 12, seed=seed)[0].cpu().numpy()))
        mb.append(_inertia(X, MiniBatchKMeans(n_clusters=12, batch_size=4096, max_iter=5000, random_state=seed).fit_predict(X)))
        full.append(_inertia(X, KMeans(n_clusters=12, n_init=1, random_state=seed).fit_predict(X)))
    print(f"median inertia: device {np.median(ours):.1f}, MiniBatchKMeans {np.median(mb):.1f}, KMeans {np.median(full):.1f}")
    assert np.median(ours) <= 1.02 * np.median(mb)
    assert np.median(ours) <= 1.02 * np.median(full)


@pytest.mark.parametrize("M,dims,k", [(50000, 32, 21), (8000, 384, 20), (6000, 768, 64), (9000, 64, 256)])
def test_kmeans_is_bit_reproducible(cuda, M, dims, k):
    cluster = load_pkg("cluster")
    X, _ = _planted(M + dims, M, dims, max(2, k // 2), 1.0, 0.5)
    Xd = torch.from_numpy(X).to(cuda)
    a = cluster.kmeans(Xd, k, seed=7)
    b = cluster.kmeans(Xd, k, seed=7)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    lab = a[0].cpu().numpy()
    assert lab.min() >= 0 and lab.max() < k
    assert torch.isfinite(a[1]).all()


def test_semantic_chain_from_images(cuda, tmp_path):
    """extract_all (multi-region) -> extract_bboxes -> extract_bbox_features -> extract_bbox_clusters ->
    extract_semantic_segmentations on synthetic images with seeded weights."""
    import cv2
    from oracle import bbox_ref
    ex = load_pkg("extract"); synth = load_pkg("synth")
    root = tmp_path / "images"
    root.mkdir()
    names = []
    for i in range(8):
        img = synth.blobs_image(160, 208, 40 + i).numpy()
        names.append(f"im{i:03d}.jpg")
        cv2.imwrite(str(root / names[-1]), cv2.cvtColor(img, cv2.COLOR_RGB2BGR), [cv2.IMWRITE_JPEG_QUALITY, 95])
    (tmp_path / "list.txt").write_text("\n".join(names) + "\n")
    fdir, edir, mdir = tmp_path / "features", tmp_path / "eigs", tmp_path / "multi"
    ex.extract_all(str(tmp_path / "list.txt"), str(root), "dino_vits16", str(fdir), str(edir), K=5, batch_size=4, seed=0,
                   multi_region_dir=str(mdir), non_adaptive_num_segments=4)
    ex.extract_bboxes(str(fdir), str(mdir), str(tmp_path / "bboxes.pth"), num_erode=2, num_dilate=3)
    boxes = torch.load(tmp_path / "bboxes.pth", weights_only=False)
    for d in boxes:
        m = np.array(Image.open(mdir / f"{d['id']}.png"))
        assert np.array_equal(_rows(d), _rows(bbox_ref.extract_bbox(m, d["id"], 16, 2, 3, True)))
    ex.extract_bbox_features(str(root), str(tmp_path / "bboxes.pth"), "dino_vits16", str(tmp_path / "feats.pth"), seed=0)
    ex.extract_bbox_clusters(str(tmp_path / "feats.pth"), str(tmp_path / "clusters.pth"), num_clusters=3, seed=0, pca_dim=4)
    clusters = torch.load(tmp_path / "clusters.pth", weights_only=False)
    for d in clusters:
        assert "features" not in d
        assert d["clusters"].dtype == np.int32 and len(d["clusters"]) == len(d["bboxes"])
        assert ((d["clusters"] >= 0) & (d["clusters"] < 3)).all()
    sem = tmp_path / "semantic"
    ex.extract_semantic_segmentations(str(mdir), str(tmp_path / "clusters.pth"), str(sem))
    for d in clusters:
        m = np.array(Image.open(mdir / f"{d['id']}.png"))
        lut = np.zeros(256, np.int64)
        lut[np.array(d["segment_indices"], np.int64)] = d["clusters"]
        assert np.array_equal(np.array(Image.open(sem / f"{d['id']}.png")), lut[m].astype(np.uint8))
