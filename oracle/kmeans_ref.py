"""ORACLE (test infrastructure, not product): float64 restatement of the two device K-means kernels,
``dss_segment_kmeans`` (csrc/segment.cu) and ``dss_kmeans`` (csrc/cluster.cu), step for step.

Both kernels run scikit-learn's algorithm -- greedy k-means++ seeding (``sklearn.cluster.kmeans_plusplus``) and
``_kmeans_single_lloyd`` -- with numpy's RNG replaced by a counter-based hash. This module holds:

- ``seg_uniform``: a bit-exact port of ``seg_hash`` / ``seg_uniform`` (csrc/kmeans_common.cuh). Counter 0 picks the
  first centre as ``min(M - 1, floor(u * M))``; counter ``1 + (c - 1) * trials + t`` is local trial t of centre c.
  ``dss_kmeans`` uses key 0, ``dss_segment_kmeans`` the image key (or the batch position).
- ``CounterRandomState``: a ``np.random.RandomState`` whose ``choice`` and ``uniform`` hand out that stream, so that
  scikit-learn's own ``kmeans_plusplus`` picks the seeds the kernels should pick.
- ``seed_indices`` / ``lloyd``: numpy restatements of the two phases, proven equal to scikit-learn on the CPU
  (tests/test_cpu_kmeans_ref.py), that also report the decision margins a float32 kernel has to clear to make the same
  choices. Distances are computed directly as sum (x - c)^2, so integer-valued data stays exact.
- ``segment_labels``: the background swap of the multi-region segmentation on top of the labels.

Only tests/ may import this module."""
from __future__ import annotations

import numpy as np

from .segment_ref import get_border_fraction

_MASK = 0xFFFFFFFF


def seg_hash(a: int, b: int, c: int) -> int:
    """csrc/kmeans_common.cuh seg_hash, with 32-bit wrap-around."""
    x = ((a * 0x9E3779B1) & _MASK) ^ ((((b + 0x7F4A7C15) & _MASK) * 0x85EBCA77) & _MASK) ^ \
        ((((c + 0x165667B1) & _MASK) * 0xC2B2AE3D) & _MASK)
    x ^= x >> 16
    x = (x * 0x7FEB352D) & _MASK
    x ^= x >> 15
    x = (x * 0x846CA68B) & _MASK
    x ^= x >> 16
    return x


def seg_uniform(seed: int, key: int, ctr: int) -> float:
    """Uniform in [0, 1) with 24 random bits, keyed by (seed, stream key, counter)."""
    return (seg_hash(seed & _MASK, key & _MASK, ctr & _MASK) >> 8) * (1.0 / 16777216.0)


def local_trials(k: int) -> int:
    return 2 + int(np.log(k))


class CounterRandomState(np.random.RandomState):
    """A RandomState whose ``choice`` and ``uniform`` return the kernels' counter stream in order (counter 0, 1, ...).
    ``choice(n)`` maps u to ``min(n - 1, floor(u * n))``; its weights must be uniform (scikit-learn passes
    sample_weight / sum, all equal without sample weights)."""

    def __init__(self, seed: int, key: int = 0):
        super().__init__(0)
        self.stream_seed, self.stream_key, self.ctr = int(seed), int(key), 0

    def _next(self) -> float:
        u = seg_uniform(self.stream_seed, self.stream_key, self.ctr)
        self.ctr += 1
        return u

    def choice(self, a, size=None, replace=True, p=None):
        n = int(a) if np.isscalar(a) else len(a)
        if size is not None or (p is not None and not np.allclose(p, 1.0 / n)):
            raise NotImplementedError("CounterRandomState.choice: one draw with uniform weights only")
        i = min(n - 1, int(self._next() * n))
        return i if np.isscalar(a) else a[i]

    def uniform(self, low=0.0, high=1.0, size=None):
        if size is None:
            return low + (high - low) * self._next()
        n = int(np.prod(size))
        return low + (high - low) * np.array([self._next() for _ in range(n)]).reshape(size)


def _sqdist(X: np.ndarray, C: np.ndarray, block_elems: int = 1 << 22) -> np.ndarray:
    """[M, k] squared distances sum_j (x_j - c_j)^2 in float64, in row blocks."""
    M, d = X.shape
    k = C.shape[0]
    rows = max(1, block_elems // max(1, k * d))
    out = np.empty((M, k))
    for r0 in range(0, M, rows):
        diff = X[r0:r0 + rows, None, :] - C[None, :, :]
        out[r0:r0 + rows] = np.einsum("mkd,mkd->mk", diff, diff)
    return out


def _boundary_margin(prefix: np.ndarray, target: float) -> float:
    """Distance of a draw target to the nearest prefix-sum boundary (0 counts as a boundary)."""
    i = np.searchsorted(prefix, target)
    near = [target]
    if i < len(prefix):
        near.append(abs(prefix[i] - target))
    if i > 0:
        near.append(abs(target - prefix[i - 1]))
    return float(min(near))


def seed_indices(X, k: int, seed: int, key: int = 0) -> dict:
    """Greedy k-means++ (sklearn _kmeans_plusplus) driven by the counter stream: the candidate of a target u * pot is
    the first point whose inclusive prefix sum of the squared distances reaches it; the candidate with the smallest
    potential wins (ties -> the lower trial). Returns the chosen row indices and the decision margins:
    draw_margin[i] = distance of each target to the nearest prefix boundary, divided by the target;
    trial_gap[i] = (second-best - best) / best over the trials whose candidate differs from the best one's (inf if none)."""
    X = np.asarray(X, np.float64)
    M = X.shape[0]
    trials = local_trials(k)
    first = min(M - 1, int(seg_uniform(seed, key, 0) * M))
    idx = [first]
    closest = _sqdist(X, X[first:first + 1])[:, 0]
    pot = closest.sum()
    draw_margin, trial_gap = [], []
    for c in range(1, k):
        targets = np.array([seg_uniform(seed, key, 1 + (c - 1) * trials + t) for t in range(trials)]) * pot
        prefix = np.cumsum(closest)
        cand = np.minimum(np.searchsorted(prefix, targets), M - 1)
        for t in targets:
            draw_margin.append(_boundary_margin(prefix, t) / t if t > 0 else 0.0)
        dist = np.minimum(closest[None, :], _sqdist(X, X[cand]).T)
        pots = dist.sum(axis=1)
        best = int(np.argmin(pots))
        others = pots[cand != cand[best]]
        trial_gap.append(float((others.min() - pots[best]) / pots[best]) if len(others) and pots[best] > 0 else np.inf)
        idx.append(int(cand[best]))
        closest = dist[best]
        pot = pots[best]
    return {"indices": np.array(idx, np.int64), "draw_margin": np.array(draw_margin), "trial_gap": np.array(trial_gap)}


def _estep(X: np.ndarray, C: np.ndarray, gamma: float):
    """Nearest centre (ties -> lower index), its squared distance, and the E-step margin: the smallest
    (d_j - d_best) / (gamma * (d_j + d_best)) over the points and the centres j other than the best (inf for k = 1).
    A float32 kernel whose squared distances carry a relative error below gamma picks the same centres when the
    margin exceeds 1."""
    D = _sqdist(X, C)
    rows = np.arange(len(X))
    labels = np.argmin(D, axis=1)
    d1 = D[rows, labels]
    if C.shape[0] == 1:
        return labels, d1, np.inf
    with np.errstate(divide="ignore", invalid="ignore"):
        r = (D - d1[:, None]) / (gamma * (D + d1[:, None]))
    r[D == d1[:, None]] = 0.0   # exact ties
    r[rows, labels] = np.inf
    return labels, d1, float(r.min())


def _label_sums(X: np.ndarray, labels: np.ndarray, k: int):
    order = np.argsort(labels, kind="stable")
    counts = np.bincount(labels, minlength=k)
    sums = np.zeros((k, X.shape[1]))
    nz = np.flatnonzero(counts)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])[nz]
    sums[nz] = np.add.reduceat(X[order], starts, axis=0)
    return sums, counts


def lloyd(X, init, max_iter: int = 300, tol: float = 1e-4, centre_dtype=None, gamma: float = 2.0 ** -24) -> dict:
    """scikit-learn's _kmeans_single_lloyd (dense, unit weights), restated:
    - the tolerance is tol * mean column variance (sklearn _tolerance);
    - labels start at -1; an iteration is an E step (nearest centre) and an M step (means);
    - empty clusters take the points farthest from their E-step centre (sklearn _relocate_empty_clusters_dense),
      the farthest first, ties -> lower index; the labels are left as the E step made them;
    - strict convergence (labels equal to the previous E step's) is checked before the centre shift against tol;
    - without strict convergence the E step is re-run so that the labels match the final centres;
    - the inertia is that of the final labels and centres.
    centre_dtype=np.float32 rounds the centres after every M step, as the kernels store them (scikit-learn keeps
    float64; None). Returns labels, centers, n_iter, converged, inertia and the margins: e_margin (one per E step, see
    _estep), relocated (iterations that relocated a cluster), far_gap (relative gap behind each relocated point),
    tol_gap (|shift - tol_abs| / tol_abs of every tol test, when tol > 0)."""
    X = np.asarray(X, np.float64)
    C = np.array(init, np.float64)
    M, d = X.shape
    k = C.shape[0]
    tol_abs = float(np.var(X, axis=0).mean() * tol) if tol else 0.0
    labels_old = np.full(M, -1)
    e_margin, relocated, far_gap, tol_gap = [], [], [], []
    strict, converged = False, False
    for i in range(max_iter):
        labels, dist, m = _estep(X, C, gamma)
        e_margin.append(m)
        sums, counts = _label_sums(X, labels, k)
        empty = np.flatnonzero(counts == 0)
        if len(empty):
            order = np.argsort(-dist, kind="stable")
            for c, f in zip(empty, order[:len(empty)]):
                old = labels[f]
                sums[old] -= X[f]
                counts[old] -= 1
                sums[c] = X[f]
                counts[c] = 1
            nxt = dist[order[len(empty)]] if len(order) > len(empty) else 0.0
            far_gap.append(float((dist[order[len(empty) - 1]] - nxt) / max(dist[order[0]], 1e-300)))
            relocated.append(i)
        newC = np.where(counts[:, None] > 0, sums / np.maximum(counts, 1)[:, None], C)
        if centre_dtype is not None:
            newC = newC.astype(centre_dtype).astype(np.float64)
        shift = float(((newC - C) ** 2).sum())
        C = newC
        if np.array_equal(labels, labels_old):
            strict = converged = True
            break
        if tol_abs > 0:
            tol_gap.append(abs(shift - tol_abs) / tol_abs)
        if shift <= tol_abs:
            converged = True
            break
        labels_old = labels
    if not strict:
        labels, dist, m = _estep(X, C, gamma)
        e_margin.append(m)
    inertia = float(((X - C[labels]) ** 2).sum())
    return {"labels": labels, "centers": C, "n_iter": i + 1, "converged": converged, "inertia": inertia,
            "tol_abs": tol_abs, "e_margin": np.array(e_margin), "relocated": relocated, "far_gap": np.array(far_gap),
            "tol_gap": np.array(tol_gap)}


def segment_labels(labels: np.ndarray, grid_h: int, grid_w: int) -> np.ndarray:
    """Background swap of the multi-region segmentation (extract.py:337-345): the label with the largest border share
    (ties -> the smallest label) trades places with label 0."""
    segmap = np.asarray(labels).reshape(grid_h, grid_w).copy()
    indices, fractions = get_border_fraction(segmap)
    bg = indices[np.argmax(fractions)].item()
    bg_region, zero_region = segmap == bg, segmap == 0
    segmap[bg_region] = 0
    segmap[zero_region] = bg
    return segmap.reshape(-1)
