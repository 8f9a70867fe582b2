"""-m gpu: both K-means kernels step for step against the float64 oracle (oracle/kmeans_ref.py, itself checked against
scikit-learn in tests/test_cpu_kmeans_ref.py), driven by the kernels' own counter-based random stream.

Exactness is decided by construction. The data are integer-valued (|x| <= 64, dims < 1024), so every squared distance
to a data point is an integer below 2^24 and every D^2 prefix sum and trial potential is exact on both sides: the
seeding and the first E step must agree exactly, ties included. The M step is exact in the kernels' fixed-point (cluster)
and fp64 (segment) sums, so the device centres equal the oracle's means rounded to float32 bit for bit. From the second
E step on, the centres are not integers, and each test asserts that the oracle's decision margins clear the float32
error bound of the kernels' distances (relative gamma = (dims + 8) 2^-24), so a fixture that stops being decidable
fails loudly instead of flaking. Also: covariance and PCA projection against float64 numpy at tile and split edges."""
import numpy as np
import pytest
import torch

from conftest import load_pkg
from oracle import kmeans_ref as kr

pytestmark = pytest.mark.gpu


def _int_mixture(seed, M, dims, k_true, spread=24.0, noise=4.0):
    g = np.random.default_rng(seed)
    centres = g.normal(size=(k_true, dims)) * spread
    X = centres[g.integers(0, k_true, M)] + g.normal(size=(M, dims)) * noise
    # + 0.0 turns rint's -0.0 into +0.0: the fixed-point centre sums return +0.0, and centres are compared bitwise
    return (np.clip(np.rint(X), -64, 64) + 0.0).astype(np.float32)


def _gamma(dims):
    return (dims + 8) * 2.0 ** -24


def _oracle(X, k, seed, key, max_iter, tol):
    """Seeds and trajectory of the kernels, and the assertion that they are decidable in float32."""
    s = kr.seed_indices(X, k, seed, key)
    assert s["draw_margin"].min(initial=1.0) > 2.0 ** -40, "a D^2 draw lands on a prefix boundary"
    o = kr.lloyd(X, X[s["indices"]].astype(np.float64), max_iter, tol, centre_dtype=np.float32,
                 gamma=_gamma(X.shape[1]))
    # the first E step is exact (integer centres); the later ones must clear the float32 bound
    assert o["e_margin"][1:].min(initial=np.inf) > 1.0, f"E-step margin {o['e_margin']}"
    assert o["far_gap"].min(initial=1.0) > 1e-3
    assert o["tol_gap"].min(initial=1.0) > 1e-4, "a centre shift lies on the tolerance"
    return s, o


# (M, dims, k, max_iter, tol): every NJ instantiation (dims 1..768), column tiles with partial last tiles
# (k=64/dims=200, k=200/dims=50, k=256/dims=64; k=64/dims=768 has six full tiles), and M at the layout edges:
# M = k, M < 512, 513, 1023 / 1025 (Gp 1 -> 2), >= 16896 (Gc = 264), >= 65536 (64 accumulation slots)
CLUSTER_CASES = [
    (1000, 1, 2, 300, 1e-4),
    (500, 1, 1, 300, 1e-4),
    (300, 31, 21, 300, 1e-4),
    (513, 33, 21, 3, 0.0),
    (1023, 64, 64, 300, 0.0),
    (1025, 100, 21, 2, 1e-4),
    (1800, 200, 64, 300, 1e-4),
    (1200, 300, 21, 300, 1e-4),
    (1100, 768, 64, 2, 1e-4),
    (64, 16, 64, 300, 1e-4),
    (2500, 50, 200, 3, 1e-4),
    (3000, 64, 256, 1, 1e-4),
    (2000, 64, 65, 2, 0.0),
    (16896, 8, 6, 300, 1e-4),
    (70000, 12, 6, 3, 1e-4),
]


@pytest.mark.parametrize("M,dims,k,max_iter,tol", CLUSTER_CASES)
def test_cluster_kmeans_follows_the_oracle(cuda, M, dims, k, max_iter, tol):
    cluster = load_pkg("cluster")
    X = _int_mixture(M * 7 + dims, M, dims, max(2, k // 2))
    seed = 3 + k
    _, o = _oracle(X, k, seed, 0, max_iter, tol)
    labels, centres, info, inertia = cluster.kmeans(torch.from_numpy(X).to(cuda), k, seed=seed, max_iter=max_iter, tol=tol)
    labels, centres, info = labels.cpu().numpy(), centres.cpu().numpy(), info.cpu().numpy()
    assert np.array_equal(labels, o["labels"])
    assert np.array_equal(centres.view(np.uint32), o["centers"].astype(np.float32).view(np.uint32))
    assert (int(info[0]), int(info[1])) == (o["n_iter"], int(o["converged"]))
    assert abs(float(inertia) - o["inertia"]) <= 1e-5 * o["inertia"]


def test_cluster_kmeans_seeding_with_a_multi_pass_chunk_scan(cuda):
    """M > 262144 points: the D^2 chunk sums are scanned in several passes of 512; max_iter = 1 pins the seeds, the
    first E step and the M step bit for bit."""
    cluster = load_pkg("cluster")
    M, dims, k = 300_000, 4, 6
    X = _int_mixture(42, M, dims, 4)
    s = kr.seed_indices(X, k, 9)
    assert s["draw_margin"].min() > 2.0 ** -40
    o = kr.lloyd(X, X[s["indices"]].astype(np.float64), 1, 1e-4, centre_dtype=np.float32, gamma=_gamma(dims))
    _, centres, info, _ = cluster.kmeans(torch.from_numpy(X).to(cuda), k, seed=9, max_iter=1)
    assert np.array_equal(centres.cpu().numpy().view(np.uint32), o["centers"].astype(np.float32).view(np.uint32))
    assert int(info[0]) == 1


@pytest.mark.parametrize("scale,spread,signs", [(1e4, 1e-2, False), (1e-4, 1e-5, True), (50.0, 30.0, True)])
def test_cluster_kmeans_centres_and_inertia_at_extreme_scales(cuda, scale, spread, signs):
    """Properties only (float32 cannot be compared exactly here): at strict convergence every device centre is the
    float64 mean of the points the device labelled with it, to float32 rounding of the data scale, and the inertia is
    the sum of the squared distances to the nearest device centre. Exercises the fixed-point scale at its limits."""
    cluster = load_pkg("cluster")
    g = np.random.default_rng(int(scale * 1e6) % 1000)
    M, dims, k = 20000, 24, 12
    base = g.normal(size=(k, dims)) * spread * 4
    offs = (g.choice([-1.0, 1.0], size=dims) if signs else np.ones(dims)) * scale
    X = (offs + base[g.integers(0, k, M)] + g.normal(size=(M, dims)) * spread).astype(np.float32)
    labels, centres, info, inertia = cluster.kmeans(torch.from_numpy(X).to(cuda), k, seed=1, max_iter=300, tol=0.0)
    labels, C = labels.cpu().numpy(), centres.cpu().numpy().astype(np.float64)
    assert int(info[1]) == 1
    X64 = X.astype(np.float64)
    ulp = 2.0 ** -23 * np.abs(X64).max(0)
    for c in range(k):
        pts = X64[labels == c]
        assert len(pts) > 0
        assert np.all(np.abs(C[c] - pts.mean(0)) <= 2 * ulp), c
    d2 = kr._sqdist(X64, C)
    assert np.array_equal(np.argmin(d2, 1)[d2.min(1) < np.partition(d2, 1, 1)[:, 1] * (1 - 1e-4)],
                          labels[d2.min(1) < np.partition(d2, 1, 1)[:, 1] * (1 - 1e-4)])
    want = d2[np.arange(M), labels].sum()
    assert abs(float(inertia) - want) <= 1e-4 * want


# ------------------------------------------------------------------------------------------- per-image k-means
GRID = (23, 31)


def _segment_batch(seed, B, dims, ks):
    N = GRID[0] * GRID[1]
    X = np.stack([_int_mixture(seed * 1000 + b, N, dims, ks[b], spread=30.0, noise=3.0) for b in range(B)])
    return X


@pytest.mark.parametrize("max_iter,tol", [(1, 1e-4), (2, 0.0), (3, 1e-4), (300, 1e-4), (300, 0.0)])
@pytest.mark.parametrize("layout,keys,infer_bg", [("eigenvectors", True, True), ("features", False, False),
                                                  ("features", True, True)])
def test_segment_kmeans_follows_the_oracle(cuda, max_iter, tol, layout, keys, infer_bg):
    """B = 300 images (more than 2 x 132 CTAs: CTAs are reused), per-image k, with and without image keys, both point
    layouts (the eigenvector layout is the strided view evecs[:, 1:1+m]), the background swap on a 23 x 31 grid."""
    segment = load_pkg("segment")
    B, dims, seed = 300, 4, 5
    g = np.random.default_rng(17)
    ks = [int(x) for x in g.integers(2, 9, size=B)]
    X = _segment_batch(3, B, dims, ks)                           # [B, N, dims]
    image_keys = [int(x) for x in g.integers(0, 1 << 31, size=B)] if keys else None
    if layout == "eigenvectors":
        evecs = np.zeros((B, dims + 2, X.shape[1]), np.float32)   # row 0 and the last row are not used
        evecs[:, 1:1 + dims] = X.transpose(0, 2, 1)
        pts = torch.from_numpy(evecs).to(cuda)[:, 1:1 + dims]
    else:
        pts = torch.from_numpy(X).to(cuda)
    labels, info, inertia = segment.kmeans_labels(pts, ks, grid=GRID if infer_bg else None, infer_bg_index=infer_bg,
                                                  layout=layout, seed=seed, max_iter=max_iter, tol=tol,
                                                  image_keys=image_keys)
    labels, info, inertia = labels.cpu().numpy(), info.cpu().numpy(), inertia.cpu().numpy()
    for b in range(B):
        key = image_keys[b] if keys else b
        _, o = _oracle(X[b], ks[b], seed, key, max_iter, tol)
        want = kr.segment_labels(o["labels"], *GRID) if infer_bg else o["labels"]
        assert np.array_equal(labels[b], want), b
        assert (int(info[b, 0]), int(info[b, 1])) == (o["n_iter"], int(o["converged"])), b
        assert abs(float(inertia[b]) - o["inertia"]) <= 1e-5 * o["inertia"], b


def test_segment_kmeans_key_changes_the_stream(cuda):
    segment = load_pkg("segment")
    X = _segment_batch(4, 2, 3, [6, 6])
    pts = torch.from_numpy(np.stack([X[0], X[0]])).to(cuda)
    labels, _, _ = segment.kmeans_labels(pts, 6, layout="features", seed=1, max_iter=1, image_keys=[5, 6])
    labels = labels.cpu().numpy()
    for b, key in enumerate((5, 6)):
        _, o = _oracle(X[0], 6, 1, key, 1, 1e-4)
        assert np.array_equal(labels[b], o["labels"])
    assert not np.array_equal(kr.seed_indices(X[0], 6, 1, 5)["indices"], kr.seed_indices(X[0], 6, 1, 6)["indices"])


# --------------------------------------------------------------------------------------------- covariance / PCA
@pytest.mark.parametrize("d", [1, 5, 100, 1000, 1024])
@pytest.mark.parametrize("M", [2, 3, 31, 33, 17000])
def test_covariance_at_tile_and_split_edges(cuda, M, d):
    if M * d > 17000 * 100 and M > 33:
        M = 2000                      # keeps the float64 reference cheap at d = 1000 / 1024
    cluster = load_pkg("cluster")
    g = np.random.default_rng(M * 7 + d)
    X = (g.normal(size=(M, d)) * np.linspace(0.5, 3.0, d) + g.normal(size=d)).astype(np.float32)
    mean, cov = cluster.covariance(torch.from_numpy(X).to(cuda))
    x64 = X.astype(np.float64)
    want = np.atleast_2d(np.cov(x64, rowvar=False))
    got = cov[:, :d].double().cpu().numpy()
    scale = np.sqrt(np.outer(np.diag(want), np.diag(want))) + 1e-30
    assert np.abs(got - want).max() <= 1e-6 * scale.max()
    assert np.abs(mean.double().cpu().numpy() - x64.mean(0)).max() <= 1e-6 * np.abs(x64).max()
    assert torch.equal(cov[:, d:].cpu(), torch.zeros(d, cov.shape[1] - d))
    assert np.array_equal(got, got.T)


@pytest.mark.parametrize("d", [5, 33, 100, 1000])
@pytest.mark.parametrize("p", [1, 3, 17, 64])
def test_pca_project_matches_float64(cuda, d, p):
    cluster = load_pkg("cluster")
    g = np.random.default_rng(d * 100 + p)
    M = 1000 + 37                                   # not a multiple of 64
    X = (g.normal(size=(M, d)) + 0.5).astype(np.float32)
    mean = X.mean(0).astype(np.float32)
    V = g.normal(size=(p, d)).astype(np.float32)
    Y = cluster.pca_project(torch.from_numpy(X).to(cuda), torch.from_numpy(mean).to(cuda),
                            torch.from_numpy(V).to(cuda)).cpu().numpy()
    C = X.astype(np.float64) - mean.astype(np.float32).astype(np.float64)
    want = C @ V.astype(np.float64).T
    bound = 4 * d * 2.0 ** -24 * (np.abs(C) @ np.abs(V.astype(np.float64)).T) + 1e-30
    assert Y.shape == (M, p)
    assert np.all(np.abs(Y - want) <= bound)
