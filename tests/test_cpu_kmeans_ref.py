"""The float64 K-means oracle (oracle/kmeans_ref.py) against scikit-learn itself: the counter-stream k-means++ seeding
against sklearn.cluster.kmeans_plusplus driven by a CounterRandomState, and the Lloyd restatement against
KMeans(init=..., n_init=1, algorithm="lloyd") over the max_iter / tol matrix, including an empty-cluster relocation.
Continuous data: scikit-learn centres X and uses ||x||^2 - 2 x.c + ||c||^2, which can break the exact ties integer
data would create."""
import numpy as np
import pytest

from oracle import kmeans_ref as kr


def test_seg_uniform_stream_is_24_bit_and_keyed():
    u = [kr.seg_uniform(3, 5, c) for c in range(2000)]
    assert all(0.0 <= x < 1.0 and (x * 16777216.0).is_integer() for x in u)
    assert len(set(u)) > 1990
    assert kr.seg_uniform(3, 6, 0) != kr.seg_uniform(3, 5, 0) != kr.seg_uniform(4, 5, 0)
    # wrap-around: keys and counters are taken mod 2^32
    assert kr.seg_uniform(3, 5 + (1 << 32), 7) == kr.seg_uniform(3, 5, 7)
    assert kr.local_trials(1) == 2 and kr.local_trials(21) == 5 and kr.local_trials(256) == 7


def _mixture(rng, M, d, k):
    centres = rng.normal(size=(k, d)) * rng.uniform(1.0, 4.0)
    return centres[rng.integers(0, k, M)] + rng.normal(size=(M, d)) * rng.uniform(0.5, 3.0, size=d)


@pytest.mark.parametrize("case", range(20))
def test_seeding_equals_sklearn_kmeans_plusplus(case):
    from sklearn.cluster import kmeans_plusplus
    rng = np.random.default_rng(100 + case)
    k = [1, 2, 3, 5, 8, 13, 21, 40, 64, 65, 100, 128, 200, 256][case % 14]
    M = int(rng.integers(k, 4 * k + 400))
    d = int(rng.integers(1, 48))
    X = _mixture(rng, M, d, max(1, k // 3))
    seed, key = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 31))
    got = kr.seed_indices(X, k, seed, key)
    _, want = kmeans_plusplus(X, k, random_state=kr.CounterRandomState(seed, key))
    assert np.array_equal(got["indices"], want)
    assert len(set(want.tolist())) == k


def _lloyd_cases():
    for case in range(4):
        for max_iter in (1, 2, 3, 300):
            for tol in (0.0, 1e-4):
                yield case, max_iter, tol


@pytest.mark.parametrize("case,max_iter,tol", list(_lloyd_cases()))
def test_lloyd_equals_sklearn(case, max_iter, tol):
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(case)
    M, d, k = [(1500, 5, 8), (800, 1, 4), (2000, 17, 21), (600, 33, 3)][case]
    X = _mixture(rng, M, d, max(2, k - 2))          # fewer true clusters than k: several iterations
    init = X[kr.seed_indices(X, k, case)["indices"]]
    o = kr.lloyd(X, init, max_iter, tol)
    km = KMeans(k, init=init, n_init=1, algorithm="lloyd", max_iter=max_iter, tol=tol).fit(X)
    assert np.array_equal(o["labels"], km.labels_)
    assert o["n_iter"] == km.n_iter_
    assert np.allclose(o["centers"], km.cluster_centers_, rtol=1e-10, atol=1e-10 * np.abs(X).max())
    assert abs(o["inertia"] - km.inertia_) <= 1e-10 * km.inertia_
    if o["n_iter"] < max_iter:
        assert o["converged"]


def test_lloyd_reaches_the_cap_and_converges_with_sklearn():
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(7)
    X = _mixture(rng, 3000, 6, 5)
    init = X[kr.seed_indices(X, 12, 1)["indices"]]
    full = kr.lloyd(X, init, 300, 0.0)
    assert full["converged"] and full["n_iter"] > 4
    capped = kr.lloyd(X, init, full["n_iter"] - 2, 0.0)
    assert not capped["converged"] and capped["n_iter"] == full["n_iter"] - 2
    km = KMeans(12, init=init, n_init=1, algorithm="lloyd", max_iter=full["n_iter"] - 2, tol=0.0).fit(X)
    assert np.array_equal(capped["labels"], km.labels_)   # labels re-assigned to the final centres at the cap
    assert abs(capped["inertia"] - km.inertia_) <= 1e-10 * km.inertia_


@pytest.mark.parametrize("max_iter,tol", [(1, 0.0), (2, 1e-4), (300, 1e-4), (300, 0.0)])
def test_lloyd_relocates_one_empty_cluster_like_sklearn(max_iter, tol):
    """One initial centre lies far from every point: its cluster is empty after the first E step and takes the point
    farthest from its centre; the labels are left as the E step made them."""
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(11)
    X = _mixture(rng, 900, 3, 4)
    init = X[kr.seed_indices(X, 5, 2)["indices"]].copy()
    init[3] = X.max(0) + 50.0
    o = kr.lloyd(X, init, max_iter, tol)
    assert o["relocated"][:1] == [0] and o["far_gap"][0] > 1e-6
    km = KMeans(5, init=init, n_init=1, algorithm="lloyd", max_iter=max_iter, tol=tol).fit(X)
    assert np.array_equal(o["labels"], km.labels_)
    assert o["n_iter"] == km.n_iter_
    assert np.allclose(o["centers"], km.cluster_centers_, rtol=1e-10, atol=1e-10 * np.abs(X).max())
    assert abs(o["inertia"] - km.inertia_) <= 1e-10 * km.inertia_


def test_segment_labels_swaps_the_border_label_to_zero():
    from oracle.segment_ref import get_border_fraction
    rng = np.random.default_rng(5)
    lab = rng.integers(0, 4, size=23 * 31)
    lab.reshape(23, 31)[0, :] = 2
    out = kr.segment_labels(lab, 23, 31).reshape(23, 31)
    idx, frac = get_border_fraction(lab.reshape(23, 31))
    bg = idx[np.argmax(frac)]
    assert bg == 2
    assert np.array_equal(out == 0, lab.reshape(23, 31) == 2)
    assert np.array_equal(out == 2, lab.reshape(23, 31) == 0)
