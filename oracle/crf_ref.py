"""ORACLE (test infrastructure, not product): float64 restatement of the dense CRF that the reference calls through
SimpleCRF (``denseCRF.densecrf``, extract/extract.py:688-690), and of the label upsampling around it.

SimpleCRF wraps Kraehenbuehl's densecrf; neither is installed, so the model is restated from the papers
(Kraehenbuehl & Koltun 2011; Adams, Baek & Davis 2010 for the permutohedral lattice) with densecrf's defaults, Potts
compatibility and symmetric normalisation:

    L(v)    permutohedral filter: elevate with scale sqrt(2/3)(d+1)/sqrt((i+1)(i+2)) on feature i, splat with
            barycentric weights, blur [1/2, 1, 1/2] along the d+1 lattice directions in order (missing neighbour = 0),
            slice, times 1/(1 + 2^-d)
    K~ Q    n * L(n * Q),  n = 1/sqrt(L(1) + 1e-20)
    -U      log(clip(P, eps, 1)) for the probability map P the reference builds (a one-hot map)
    Q0      softmax(-U);  Q <- softmax(-U + w1 K~bil Q + w2 K~sp Q), `it` times;  labels = argmax Q (first wins)

The embedding repeats the CUDA kernel's float64 operations one for one (numpy does not contract into FMAs), so lattice
keys, point counts and weights are bit-identical to csrc/crf.cu. ``exact_filter`` is the dense Gaussian sum the lattice
approximates. ``denseCRF`` below is a stand-in module whose ``densecrf`` runs ``mean_field``; installed in
``sys.modules`` it lets the reference's own ``_extract_crf_segmentations`` run (oracle/make_crf_golden.py)."""
from __future__ import annotations

import math
import types

import numpy as np

UNARY_EPS = 1e-5
U32 = 2.0 ** -24          # unit roundoff of fp32


# ---------------------------------------------------------------------------------------------------- label upsampling
def nn_index(dst: int, src: int) -> np.ndarray:
    """cv2.resize(INTER_NEAREST) source index of every destination index: min(floor(x * (1 / (dst / src))), src - 1)."""
    ifx = 1.0 / (float(dst) / float(src))
    return np.minimum(np.floor(np.arange(dst, dtype=np.float64) * ifx).astype(np.int64), src - 1)


def upsample_labels(segmap: np.ndarray, H: int, W: int, P: int) -> np.ndarray:
    """extract.py:673-681: the (H_pad, W_pad) nearest resize inside the patch-multiple block, the (H, W) one elsewhere."""
    sh, sw = segmap.shape
    Hp, Wp = H // P * P, W // P * P
    out = segmap[np.ix_(nn_index(H, sh), nn_index(W, sw))]
    out[:Hp, :Wp] = segmap[np.ix_(nn_index(Hp, sh), nn_index(Wp, sw))]
    return out


# ---------------------------------------------------------------------------------------------------- lattice
def scales(d: int):
    return [math.sqrt(2.0 / 3.0) * (d + 1) / math.sqrt(float((i + 1) * (i + 2))) for i in range(d)]


def key_bits(d: int, flo, fhi, B: int):
    """Bits of a lattice key as csrc/crf.cu's key_layout sizes them for features f_k in [flo_k, fhi_k] and B images:
    each coordinate field spans the interval bounds of its elevated coordinate widened by 3(d+1) + 1, the image index
    takes ceil(log2 B) bits above them. None when one field alone needs more than 62 bits or the bounds are not finite;
    the library accepts a layout iff this is <= 64. The double arithmetic repeats key_layout's order."""
    sc = scales(d)
    flo, fhi = [float(x) for x in flo], [float(x) for x in fhi]
    if not all(math.isfinite(a) and math.isfinite(b) and a <= b for a, b in zip(flo, fhi)):
        return None
    clo = [flo[k] * sc[k] for k in range(d)]
    chi = [fhi[k] * sc[k] for k in range(d)]
    total = 0
    while (1 << total) < B:
        total += 1
    for c in range(d):
        lo = hi = 0.0
        for k in range(c, d):
            lo += clo[k]
            hi += chi[k]
        if c > 0:
            lo -= c * chi[c - 1]
            hi -= c * clo[c - 1]
        margin = 3.0 * (d + 1) + 1.0
        if not (abs(lo) < 1e15 and abs(hi) < 1e15):
            return None
        span = math.ceil(hi + margin) - math.floor(lo - margin)
        w = 1
        while w < 62 and (1 << w) <= span:
            w += 1
        if (1 << w) <= span:
            return None
        total += w
    return total


def crf_key_bits(H: int, W: int, B: int, alpha: float, beta: float, gamma: float):
    """(bilateral, spatial) key bits of a dss_crf_segment call on B images of at most H x W pixels."""
    bil = key_bits(5, [0.0] * 5, [(W - 1) / alpha, (H - 1) / alpha, 255.0 / beta, 255.0 / beta, 255.0 / beta], B)
    sp = key_bits(2, [0.0] * 2, [(W - 1) / gamma, (H - 1) / gamma], B)
    return bil, sp


def embed(features: np.ndarray):
    """features [N, d] float64 -> (keys [N, d+1, d] int64 simplex vertices, weights [N, d+1] float64)."""
    f = np.asarray(features, np.float64)
    N, d = f.shape
    sc = scales(d)
    el = np.empty((N, d + 1))
    sm = np.zeros(N)
    for j in range(d, 0, -1):
        cf = f[:, j - 1] * sc[j - 1]
        el[:, j] = sm - float(j) * cf
        sm = sm + cf
    el[:, 0] = sm
    down = 1.0 / (d + 1)
    v = el * down
    up = np.ceil(v) * float(d + 1)
    dn = np.floor(v) * float(d + 1)
    rem0 = np.where(up - el < el - dn, up, dn).astype(np.int64)
    s = rem0.sum(1) // (d + 1)
    rank = np.zeros((N, d + 1), np.int64)
    for i in range(d):
        for j in range(i + 1, d + 1):
            c = (el[:, i] - rem0[:, i]) < (el[:, j] - rem0[:, j])
            rank[:, i] += c
            rank[:, j] += ~c
    sc_ = s[:, None]
    pos, neg = s > 0, s < 0
    m = (rank >= (d + 1) - sc_) & pos[:, None]
    rem0 -= (d + 1) * m
    rank += np.where(m, sc_ - (d + 1), np.where(pos[:, None], sc_, 0))
    m = (rank < -sc_) & neg[:, None]
    rem0 += (d + 1) * m
    rank += np.where(m, (d + 1) + sc_, np.where(neg[:, None], sc_, 0))
    bary = np.zeros((N, d + 2))
    ar = np.arange(N)
    for i in range(d + 1):
        vv = (el[:, i] - rem0[:, i]) * down
        bary[ar, d - rank[:, i]] = bary[ar, d - rank[:, i]] + vv
        bary[ar, d + 1 - rank[:, i]] = bary[ar, d + 1 - rank[:, i]] - vv
    bary[:, 0] = bary[:, 0] + (1.0 + bary[:, d + 1])
    keys = np.empty((N, d + 1, d), np.int64)
    for r in range(d + 1):
        keys[:, r, :] = rem0[:, :d] + np.where(rank[:, :d] <= d - r, r, r - (d + 1))
    return keys, bary[:, :d + 1]


class Lattice:
    """The permutohedral lattice of one point set; ``filter`` applies L (optionally symmetric-normalised)."""

    def __init__(self, features: np.ndarray):
        keys, self.w = embed(features)
        self.N, self.d = features.shape[0], features.shape[1]
        d = self.d
        flat = keys.reshape(-1, d)
        lo = flat.min(0) - (d + 2)
        span = flat.max(0) + (d + 2) - lo + 1
        radix = np.cumprod(np.concatenate([[1], span[::-1][:-1]]))[::-1]   # coordinate 0 most significant
        assert float(np.prod(span.astype(np.float64))) < 2.0 ** 62
        self._pack = lambda k: ((k - lo) * radix).sum(-1)
        packed = self._pack(flat)
        self.keys, self.inv = np.unique(packed, return_inverse=True)
        self.inv = self.inv.reshape(self.N, d + 1)
        self.points = len(self.keys)
        ukeys = np.unique(flat, axis=0)      # same order as self.keys (mixed radix preserves lexicographic order)
        self.nbr = []
        for k in range(d + 1):
            e = np.zeros(d, np.int64)
            if k < d:
                e[k] = d + 1
            self.nbr.append((self._find(ukeys - 1 + e), self._find(ukeys + 1 - e)))
        self._norm = None

    def _find(self, k):
        p = self._pack(k)
        i = np.searchsorted(self.keys, p)
        i = np.minimum(i, self.points - 1)
        return np.where(self.keys[i] == p, i, self.points)          # `points` = the zero row

    def apply(self, values: np.ndarray) -> np.ndarray:
        v = np.asarray(values, np.float64)
        C = v.shape[1]
        lat = np.zeros((self.points, C))
        for r in range(self.d + 1):
            for c in range(C):
                lat[:, c] += np.bincount(self.inv[:, r], weights=self.w[:, r] * v[:, c], minlength=self.points)
        for n1, n2 in self.nbr:
            z = np.vstack([lat, np.zeros((1, C))])
            lat = lat + 0.5 * (z[n1] + z[n2])
        out = np.zeros((self.N, C))
        for r in range(self.d + 1):
            out += self.w[:, r, None] * lat[self.inv[:, r]]
        return out * (1.0 / (1.0 + 2.0 ** (-self.d)))

    def norm(self) -> np.ndarray:
        if self._norm is None:
            self._norm = 1.0 / np.sqrt(self.apply(np.ones((self.N, 1)))[:, 0] + 1e-20)
        return self._norm

    def filter(self, values: np.ndarray, normalize: bool = False) -> np.ndarray:
        if not normalize:
            return self.apply(values)
        n = self.norm()[:, None]
        return n * self.apply(n * np.asarray(values, np.float64))

    def contributions(self) -> np.ndarray:
        """Number of (point, vertex) slots splatted into every lattice point."""
        return np.bincount(self.inv.ravel(), minlength=self.points)

    def _fp32_error(self, mag: np.ndarray, rel_in: np.ndarray, rel_out: np.ndarray):
        """First-order error bound of csrc/crf.cu's fp32 L on splat inputs of magnitude ``mag`` [N, C] that carry a
        relative error ``rel_in`` [N] (weights included) and an output scaling with relative error ``rel_out`` [N].
        Returns (bound, magnitude) of alpha * slice(blur(splat)), both [N, C]."""
        u, d = U32, self.d
        C = mag.shape[1]
        slots = self.inv.ravel()
        order = np.argsort(slots, kind="stable")          # the kernel's contribution order: slot index within a point
        grp = slots[order]
        pix = order // (d + 1)
        t = self.w.ravel()[order, None] * mag[pix]
        # splat, one fmaf per contribution: every partial sum is rounded once, |error| <= u sum_k |s_k|
        cum = np.cumsum(t, 0)
        first = np.searchsorted(grp, np.arange(self.points))
        base = np.vstack([np.zeros((1, C)), cum])[first][grp]
        A = np.zeros((self.points, C))
        E = np.zeros((self.points, C))
        for c in range(C):
            A[:, c] = np.bincount(grp, weights=t[:, c], minlength=self.points)
            E[:, c] = np.bincount(grp, weights=u * (cum[:, c] - base[:, c]) + rel_in[pix] * t[:, c],
                                  minlength=self.points)
        # blur, v + 0.5 (a + b): the two roundings add at most u (|v| + |a| + |b|)
        for n1, n2 in self.nbr:
            Az, Ez = np.vstack([A, np.zeros((1, C))]), np.vstack([E, np.zeros((1, C))])
            E = E + 0.5 * (Ez[n1] + Ez[n2]) + u * (A + Az[n1] + Az[n2])
            A = A + 0.5 * (Az[n1] + Az[n2])
        # slice, d + 1 fmaf with fp32 weights: (d + 2) u of the magnitude
        Eo, Ao = np.zeros((self.N, C)), np.zeros((self.N, C))
        for r in range(d + 1):
            Eo += self.w[:, r, None] * E[self.inv[:, r]]
            Ao += self.w[:, r, None] * A[self.inv[:, r]]
        alpha = 1.0 / (1.0 + 2.0 ** (-d))
        return alpha * (Eo + ((d + 2) * u + rel_out[:, None]) * Ao), alpha * Ao

    def fp32_error_bound(self, values: np.ndarray, normalize: bool = False) -> np.ndarray:
        """Componentwise bound on |dss_op_lattice_filter - filter| for fp32 ``values``, first order in u = 2^-24.

        Every fp32 operation of the kernels rounds once to nearest (no fast math), so each adds at most u times the
        magnitude of its result, and a magnitude is bounded by the same filter applied to |values|:
          - slot weights are the float64 barycentric weights rounded to fp32: u;
          - splat adds the n_j contributions of lattice point j one fmaf at a time in slot order: u sum_k |s_k| over
            its partial sums, which is where the contribution counts enter (the busiest points of a VOC-size image
            take 10^4 contributions);
          - blur pass: u (|v| + |a| + |b|); slice: (d + 2) u of the magnitude; the alpha (fp32) and output scalings
            add 2 u (3 u when normalised);
          - normalised: n = 1 / sqrtf(alpha L(1) + 1e-20) inherits half the relative error of alpha L(1) + 1e-20 (its
            alpha, product and sum roundings included) plus 2 u (sqrtf and the division), and the splat weights carry
            n (one more product).
        The neglected second-order terms are below (max_j n_j u)^2 of the bound; the float64 reference's own error is
        some 10^9 times smaller than u."""
        u = U32
        mag = np.abs(np.asarray(values, np.float64))
        one = np.full(self.N, u)
        if not normalize:
            return self._fp32_error(mag, one, 2 * one)[0] * (1 + 1e-3)
        e1, s1 = self._fp32_error(np.ones((self.N, 1)), one, 3 * one)
        en = 0.5 * (e1[:, 0] / s1[:, 0]) + 2 * u
        n = self.norm()
        e, _ = self._fp32_error(n[:, None] * mag, en + 2 * u, en + 3 * u)
        return n[:, None] * e * (1 + 1e-3)


def lattice_filter(features: np.ndarray, values: np.ndarray, normalize: bool = False) -> np.ndarray:
    return Lattice(features).filter(values, normalize)


class Exact:
    """Dense Gaussian filter sum_j exp(-|f_i - f_j|^2 / 2) v_j (the pixel itself included) in float64."""

    def __init__(self, features: np.ndarray):
        self.f = np.asarray(features, np.float64)
        self.N = self.f.shape[0]
        self._norm = None

    def apply(self, values: np.ndarray) -> np.ndarray:
        v = np.asarray(values, np.float64)
        out = np.empty((self.N, v.shape[1]))
        sq = (self.f ** 2).sum(1)
        for s in range(0, self.N, 512):
            fi = self.f[s:s + 512]
            d2 = np.maximum(sq[s:s + 512, None] + sq[None, :] - 2.0 * fi @ self.f.T, 0.0)
            out[s:s + 512] = np.exp(-0.5 * d2) @ v
        return out

    norm = Lattice.norm
    filter = Lattice.filter


def exact_filter(features: np.ndarray, values: np.ndarray, normalize: bool = False) -> np.ndarray:
    return Exact(features).filter(values, normalize)


# ---------------------------------------------------------------------------------------------------- mean field
def crf_features(image: np.ndarray, alpha: float, beta: float, gamma: float):
    """(bilateral [HW, 5], spatial [HW, 2]) features of an (H, W, 3) uint8 image, float64, x = column, y = row."""
    H, W = image.shape[:2]
    y, x = np.divmod(np.arange(H * W, dtype=np.int64), W)
    x, y = x.astype(np.float64), y.astype(np.float64)
    rgb = image.reshape(-1, 3).astype(np.float64)
    bil = np.stack([x / alpha, y / alpha, rgb[:, 0] / beta, rgb[:, 1] / beta, rgb[:, 2] / beta], 1)
    return bil, np.stack([x / gamma, y / gamma], 1)


def _softmax(l):
    e = np.exp(l - l.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def mean_field(image: np.ndarray, prob: np.ndarray, params, unary_eps: float = UNARY_EPS, filter: str = "lattice"):
    """image (H, W, 3) uint8, prob (H, W, M) the unary probability map, params (w1, alpha, beta, w2, gamma, it).
    Returns (list of Q [HW, M] after 0 .. it iterations, labels (H, W) uint8, lattice point counts (bil, sp))."""
    w1, alpha, beta, w2, gamma, it = params
    H, W = image.shape[:2]
    M = prob.shape[-1]
    neg_u = np.log(np.clip(np.asarray(prob, np.float64).reshape(H * W, M), unary_eps, 1.0))
    fb, fs = crf_features(image, float(alpha), float(beta), float(gamma))
    kind = {"lattice": Lattice, "exact": Exact}[filter]
    Kb, Ks = kind(fb), kind(fs)
    Q = _softmax(neg_u)
    Qs = [Q]
    for _ in range(int(it)):
        Q = _softmax(neg_u + float(w1) * Kb.filter(Q, True) + float(w2) * Ks.filter(Q, True))
        Qs.append(Q)
    labels = Q.argmax(1).astype(np.uint8).reshape(H, W)
    counts = (getattr(Kb, "points", 0), getattr(Ks, "points", 0))
    return Qs, labels, counts


# ---------------------------------------------------------------------------------------------------- SimpleCRF stand-in
def make_densecrf_module(unary_eps: float = UNARY_EPS, filter: str = "lattice"):
    """A module named denseCRF whose densecrf(image, unary_probabilities, params) runs mean_field; the Q of its last
    call (all iterations) and the lattice point counts are kept in ``.last``."""
    m = types.ModuleType("denseCRF")

    def densecrf(image, prob, params):
        Qs, labels, counts = mean_field(np.asarray(image), np.asarray(prob), params, unary_eps, filter)
        m.last = {"Q": Qs[-1], "counts": counts}
        return labels

    m.densecrf = densecrf
    m.last = None
    return m
