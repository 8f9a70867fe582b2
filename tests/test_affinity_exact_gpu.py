"""-m gpu: the affinity build (dss_affinity: rownorm_split_kernel, the symmetric EPI_AFFINITY_F32 GEMM epilogue,
degree_reduce_kernel) and the colour terms (dss_knn_color_counts, dss_rw_affinity_add), checked bit for bit where the
inputs make every rounding exact, and against float64 with a bound derived from where the kernel rounds otherwise.

Integer features (section 1): small integers, pre-scaled by a power of two, are exact in fp16 (lo = 0) and every
product and partial sum of the Gram matrix is an integer below 2^24, exact in any order. Under NORMALIZE the rows have
power-of-two norms (k in {1, 4, 16, 64} entries of +-2^s), so F.normalize is exact too. The float64 Gram matrix is then
THE answer: W = fp32(relu?(G) [/ max diag G] + lambda counts) with a dyadic lambda, compared with torch.equal; the
division must be the correctly rounded IEEE quotient (divisors with 21..24-bit significands).

Split terms (section 2): x = hi + lo with hi on a coarse dyadic grid and lo a few steps of a fine one, chosen so that
fp16(x) = hi, 64 lo and hi / 64 are exact normal fp16 values and hi.hi' + hi.lo' + lo.hi' fits in 24 bits: W must be
exactly that float64 sum (lo.lo' is dropped by design).

Real-valued features (sections 3, 4): per element |W - W64| <= the bound of _bound64 (split residual, fp16
underflow, 2 ulps of the running sum per wgmma k-step, normalisation and max roundings). The fp32 product that the
reference computes (torch, TF32 off) is measured against the same float64 W and printed next to the kernel's error.

Every W buffer is NaN-filled and followed by a sentinel guard image, every degree buffer likewise; the workspace is
followed by sentinel bytes. Every case checks W[:, :, :N] == its transpose bit for bit and pad columns == 0."""
import math

import numpy as np
import pytest
import scipy.sparse
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

NORMALIZE, THRESHOLD, NO_MAX = 1, 2, 4
U = 2.0 ** -24             # fp32 unit roundoff
SENT = -7777.25
WS_SLACK, WS_SENT = 1 << 20, 0xA5
N_LIST = [1, 2, 3, 5, 63, 64, 65, 127, 128, 129, 255, 256, 257, 383, 385, 713, 900, 1023, 1024, 1025]
D_LIST = [1, 8, 65, 100, 384, 768, 1024]


def _lib():
    _l = load_pkg("_lib")
    return _l, _l.load()


def _pitch(N):
    return (N + 3) // 4 * 4


def _roundup128(N):
    return (N + 127) // 128 * 128


def _cta_pairs():
    return int(_lib()[1].dss_device_sm_count()) // 2


def _items(N):
    """Work items of one image in the symmetric affinity GEMM: row-tile pair p visits the column tiles j >= 2p."""
    t = (N + 127) // 128
    return sum(max(t - 2 * p, 0) for p in range((t + 1) // 2))


def _diff(bad):
    idx = bad.nonzero()[:6].tolist()
    return f"{int(bad.sum())} of {bad.numel()} elements differ, first at {idx}"


def run_affinity(f, flags, counts=None, lam=0.0, ldw=None, degree=True):
    """dss_affinity into guarded NaN-filled buffers; checks guards, symmetry and pad columns. -> (W [B,N,ldw], deg)"""
    _l, lib = _lib()
    f = f.contiguous()
    B, N, d = f.shape
    ldw = _pitch(N) if ldw is None else ldw
    W = torch.full((B + 1, N, ldw), float("nan"), device=f.device)
    W[B] = SENT
    deg = None
    if degree:
        deg = torch.full((B + 1, N), float("nan"), device=f.device)
        deg[B] = SENT
    need = int(lib.dss_affinity_workspace_bytes(B, N, d))
    ws = torch.full((need + WS_SLACK,), WS_SENT, dtype=torch.uint8, device=f.device)
    cc = None if counts is None else counts.contiguous()
    _l.check(lib.dss_affinity(f.data_ptr(), B, N, d, flags, _l.ptr(cc), float(lam), W.data_ptr(), ldw,
                              None if deg is None else deg.data_ptr(), ws.data_ptr(), need, _l.stream_ptr()),
             "dss_affinity")
    torch.cuda.synchronize()
    assert torch.equal(W[B], torch.full_like(W[B], SENT)), "the guard image after W changed"
    assert bool((ws[need:] == WS_SENT).all()), "dss_affinity wrote past dss_affinity_workspace_bytes"
    W = W[:B]
    assert not bool(W.isnan().any()), f"elements of W left unwritten: {_diff(W.isnan())}"
    Wn = W[:, :, :N]
    assert torch.equal(Wn, Wn.transpose(1, 2)), f"W not symmetric bit for bit: {_diff(Wn != Wn.transpose(1, 2))}"
    assert bool((W[:, :, N:] == 0).all()), "pad columns [N, ldw) are not zero"
    if degree:
        assert torch.equal(deg[B], torch.full_like(deg[B], SENT)), "the guard row after degree changed"
        deg = deg[:B]
        assert not bool(deg.isnan().any()), "degree entries left unwritten"
    return W, deg


def _sym_counts(B, N, seed, dev, hi=5):
    g = torch.Generator(device=dev).manual_seed(seed)
    c = torch.randint(0, hi, (B, N, N), generator=g, device=dev, dtype=torch.uint8)
    c = torch.triu(c) + torch.triu(c, 1).transpose(1, 2)
    return c.contiguous()


# ---------------------------------------------------------------------------------------------------------------
# 1. integer features, bit for bit
def int_features(B, N, d, normalize, seed, dev, full_divisor=False):
    """Exact-arithmetic features (see the module docstring). Row 1 of every image is zero when N > 2."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rows = B * N
    if normalize:
        ks = torch.tensor([k for k in (1, 4, 16, 64) if k <= d], device=dev)
        k = ks[torch.randint(0, len(ks), (rows,), generator=g, device=dev)]
        rank = torch.rand(rows, d, generator=g, device=dev).argsort(1).argsort(1)
        sign = torch.randint(0, 2, (rows, d), generator=g, device=dev) * 2 - 1
        scale = 2.0 ** torch.randint(0, 3, (rows, 1), generator=g, device=dev)
        f = ((rank < k[:, None]) * sign * scale).float().view(B, N, d)
    else:
        f = torch.randint(-4, 5, (B, N, d), generator=g, device=dev).float()
        f[:, ::37] = 4.0                                     # hot rows
        if full_divisor:
            # one row per image with |entries| up to R, R^2 d < 2^24: max diag G is an odd integer >= 2^20
            R = min(2047, int(math.isqrt((2 ** 24 - 1) // d)))
            h = torch.randint(R // 2 + 1, R + 1, (B, d), generator=g, device=dev).float()
            h *= torch.randint(0, 2, (B, d), generator=g, device=dev) * 2 - 1
            even = (h.double().pow(2).sum(1) % 2) == 0
            h[even, 0] -= torch.sign(h[even, 0])             # flips the parity of the squared norm
            f[:, min(3, N - 1)] = h
    if N > 2:
        f[:, 1] = 0.0
    return f.contiguous()


def _epilogue64(G, flags, c, lam):
    """The reference's arithmetic on an exact float64 Gram matrix, rounded where fp32 rounds."""
    q = G.clamp_min(0.0) if flags & THRESHOLD else G
    if not flags & NO_MAX:
        mx = torch.diagonal(q, dim1=1, dim2=2).amax(1)[:, None, None]
        q = (q / mx).float().double()                    # IEEE quotient (float64 -> float32 rounding is innocuous)
    if c is not None:
        q = q + lam * c.double()
    return q.float()


def _check_degree_vs_W(deg, W, N):
    """degree against the row sums of the kernel's own W: exact when every element is a multiple of a power of two
    and the row's absolute sum stays below 2^24 of it, else within the fp32 summation bound N u sum|W|."""
    W64 = W[:, :, :N].double()
    s, a = W64.sum(2), W64.abs().sum(2)
    for unit in (1.0, 2.0 ** -2, 2.0 ** -6, 2.0 ** -8):
        if torch.equal(torch.round(W64 / unit) * unit, W64):
            if bool((a < unit * 2 ** 24).all()):
                bad = deg != s.float()
                assert not bool(bad.any()), f"degree not exact: {_diff(bad)}"
                return
            break
    err = (deg.double() - s).abs()
    assert bool((err <= N * U * a).all()), f"degree off by {(err / (N * U * a).clamp_min(1e-300)).max():.2f} x bound"


def check_exact(f, flags, counts=None, lam=0.0, degree=True, ldw=None, chunk=16):
    W, deg = run_affinity(f, flags, counts, lam, ldw, degree)
    B, N, _ = f.shape
    for z0 in range(0, B, chunk):
        z1 = min(B, z0 + chunk)
        f64 = f[z0:z1].double()
        if flags & NORMALIZE:
            f64 = f64 / f64.norm(dim=2, keepdim=True).clamp_min(1e-12)
        G = torch.bmm(f64, f64.transpose(1, 2))
        assert bool((G.abs() < 2 ** 24).all())
        want = _epilogue64(G, flags, None if counts is None else counts[z0:z1], lam)
        bad = W[z0:z1, :, :N] != want
        assert not bool(bad.any()), f"images {z0}..{z1}: {_diff(bad)}"
        if degree:
            _check_degree_vs_W(deg[z0:z1], W[z0:z1], N)
    if flags & NORMALIZE and N > 2 and counts is None:    # zero feature rows: zero row, zero column, degree 0
        assert bool((W[:, 1] == 0).all()) and (deg is None or bool((deg[:, 1] == 0).all()))
    return W, deg


@pytest.mark.parametrize("with_counts", [False, True])
@pytest.mark.parametrize("flags", range(8))
def test_integer_flags_counts_degree(cuda, flags, with_counts):
    N, d, B = 257, 100, 2
    f = int_features(B, N, d, flags & NORMALIZE, 10 + flags, cuda, full_divisor=not flags & NO_MAX)
    if not flags & (NORMALIZE | NO_MAX):
        mx = f.double().pow(2).sum(2).amax(1)
        assert bool((mx % 2 == 1).all()) and bool((mx >= 2 ** 20).all())   # divisors with full significands
    c = _sym_counts(B, N, flags, cuda) if with_counts else None
    lam = 10.0 if flags % 2 else 0.25
    W, _ = check_exact(f, flags, c, lam)
    W0, deg0 = run_affinity(f, flags, c, lam, degree=False)
    assert deg0 is None and torch.equal(W, W0), "W depends on whether the degree is requested"


@pytest.mark.parametrize("i,N", list(enumerate(N_LIST)))
def test_integer_shapes(cuda, i, N):
    d, flags = D_LIST[i % len(D_LIST)], (i * 3) % 8
    c = _sym_counts(2, N, i, cuda) if i % 3 == 0 else None
    f = int_features(2, N, d, flags & NORMALIZE, 100 + i, cuda, full_divisor=not flags & NO_MAX)
    check_exact(f, flags, c, (1.0, 10.0, 0.25)[i % 3])


@pytest.mark.parametrize("d", D_LIST)
@pytest.mark.parametrize("flags", [NORMALIZE | THRESHOLD, THRESHOLD, NO_MAX])
def test_integer_feature_dims(cuda, d, flags):
    f = int_features(1, 385, d, flags & NORMALIZE, d, cuda, full_divisor=not flags & NO_MAX)
    check_exact(f, flags)


@pytest.mark.parametrize("N,flags", [(3600, NORMALIZE | THRESHOLD), (6400, THRESHOLD)])
def test_integer_large_images(cuda, N, flags):
    """The sizes of the 480x480 and 640x640 dino_vitb8 configurations (C3 with its colour term)."""
    c = _sym_counts(1, N, N, cuda) if N == 3600 else None
    f = int_features(1, N, 384, flags & NORMALIZE, N, cuda, full_divisor=not flags & NORMALIZE)
    check_exact(f, flags, c, 10.0)


@pytest.mark.parametrize("case", ["one", "fewer_items_than_pairs", "just_more_items", "bench_264", "ragged_265"])
def test_integer_batches(cuda, case):
    pairs = _cta_pairs()
    N, d, B = {"one": (900, 384, 1), "fewer_items_than_pairs": (900, 384, max(1, (pairs - 1) // _items(900))),
               "just_more_items": (196, 384, pairs // 2 + 1), "bench_264": (900, 384, 264),
               "ragged_265": (900, 384, 265)}[case]
    items = B * _items(N)
    if case == "fewer_items_than_pairs":
        assert items < pairs
    if case == "just_more_items":
        assert pairs < items < 2 * pairs
    if case == "ragged_265":
        assert items % pairs != 0
    for flags in (NORMALIZE | THRESHOLD, THRESHOLD):
        f = int_features(B, N, d, flags & NORMALIZE, B + flags, cuda, full_divisor=not flags & NORMALIZE)
        check_exact(f, flags)


# ---------------------------------------------------------------------------------------------------------------
# 2. the three split terms, exactly
def split_features(B, N, d, seed, dev):
    """x = hi + lo: hi = +-{1, 1.5}, lo = sign(hi) j 2^-13 with j in -1..3 (below a power of two the fp16 spacing
    halves, so |lo| may only grow |x| by more than half a step). Pre-scaled by 1/2 in the kernel (max|x| in (1, 2))."""
    g = torch.Generator(device=dev).manual_seed(seed)
    sgn = (torch.randint(0, 2, (B, N, d), generator=g, device=dev) * 2 - 1).double()
    hi = sgn * (1.0 + 0.5 * torch.randint(0, 2, (B, N, d), generator=g, device=dev).double())
    lo = sgn * torch.randint(-1, 4, (B, N, d), generator=g, device=dev).double() * 2.0 ** -13
    hi[:, :, 0], lo[:, :, 0] = 1.5, 3 * 2.0 ** -13          # max|x| = 1.5 + 3 2^-13 in every image
    x = (hi + lo).float()
    assert torch.equal(x.double(), hi + lo)
    # the kernel's operands after the pre-scaling by 2^-ceil(log2 max|x|) = 1/2
    assert bool((x.abs().amax((1, 2)) > 1).all()) and bool((x.abs().amax((1, 2)) < 2).all())
    v, hv, lv = x.double() / 2, hi / 2, lo / 2
    assert torch.equal(v.half().double(), hv)                                  # fp16(x) = hi
    for t in (64 * lv, hv / 64):                                               # exact, normal (or zero) fp16
        assert torch.equal(t.half().double(), t) and bool(((t == 0) | (t.abs() >= 2.0 ** -14)).all())
    # every partial sum of hi.hi' + hi.lo' + lo.hi' is a multiple of 2^-16 (scaled units) below 2^24 of them
    sabs = d * (1.5 / 2) ** 2 + 2 * d * (1.5 / 2) * 3 * 2.0 ** -14
    assert sabs * 2 ** 16 < 2 ** 24
    return x.contiguous(), hi, lo


@pytest.mark.parametrize("B,N,d", [(2, 300, 64), (2, 300, 100), (2, 300, 384), (4, 900, 384)])
def test_split_terms_exact(cuda, B, N, d):
    x, hi, lo = split_features(B, N, d, d + N, cuda)
    for flags in (NO_MAX, NO_MAX | THRESHOLD):
        W, deg = run_affinity(x, flags)
        G = hi @ hi.transpose(1, 2) + hi @ lo.transpose(1, 2) + lo @ hi.transpose(1, 2)
        if flags & THRESHOLD:
            G = G.clamp_min(0)
        bad = W[:, :, :N] != G.float()
        assert not bool(bad.any()), _diff(bad)
        assert bool((G.float().double() == G).all())
        _check_degree_vs_W(deg, W, N)


# ---------------------------------------------------------------------------------------------------------------
# 3. real-valued features against float64
def _bound64(f, flags):
    """(W64, per-element bound) for fp32 features f [B, N, d], in the kernel's pre-scaled units (x = f 2^-e, or
    F.normalize(f)). Where the kernel rounds, per element of x (fp16 spacing 2^-11 |x|, or 2^-24 below 2^-14):
      |lo| <= L = min(|x|, max(2^-11 |x|, 2^-25)); fp16(64 lo) has error <= 2^-11 64 L + 2^-25, i.e. r = 2^-11 L + 2^-31
      on lo; fp16(hi / 64) is exact unless hi < 2^-8, else within 2^-25, which costs 2^-25 |64 lo'| = 2^-19 L' in the
      (hi/64).(64 lo') product; lo.lo' is dropped (<= L L').
    Per product: r |y| + |x| r' + 2^-19 (L + L') + L L'. Then the fp32 wgmma accumulation over 3 dpad / 16 k-steps,
    2 ulps of the running sum (<= S = sum |x||y|) per step, truncating or not; the fp32 row normalisation (rel.
    (d/32 + 10) u per row); max diag from an fp32 sum of squares ((dpad/32 + 6) u); the quotient (u |W|)."""
    B, N, d = f.shape
    dpad = (d + 63) // 64 * 64
    f64 = f.double()
    if flags & NORMALIZE:
        V = f64 / f64.norm(dim=2, keepdim=True).clamp_min(1e-12)
        e_row, unscale = (d / 32 + 10) * U, torch.ones(B, 1, 1, dtype=torch.float64, device=f.device)
    else:
        am = f.abs().amax((1, 2)).double()
        pre = torch.exp2(-torch.ceil(torch.log2(am)))[:, None, None]
        V, e_row, unscale = f64 * pre, 0.0, pre ** -2
    A = V.abs()
    S = A @ A.transpose(1, 2)
    L = torch.minimum(A, torch.clamp_min(2.0 ** -11 * A, 2.0 ** -25))
    r = 2.0 ** -11 * L + 2.0 ** -31
    T = lambda X: X.transpose(1, 2)
    Lsum = L.sum(2, keepdim=True)
    Gb = (r @ T(A) + A @ T(r) + 2.0 ** -19 * (Lsum + T(Lsum)) + L @ T(L)
          + (3 * dpad / 16 * 2.0 ** -22 + 2 * e_row) * S)
    G, Gb = (V @ V.transpose(1, 2)) * unscale, Gb * unscale
    if flags & THRESHOLD:
        G = G.clamp_min(0)
    if flags & NO_MAX:
        return G, Gb
    mx = torch.diagonal(G, dim1=1, dim2=2).amax(1)[:, None, None]
    W = G / mx
    return W, Gb / mx + W.abs() * ((dpad / 32 + 6) * U + 2 * e_row + U)


def _fp32_reference(f, flags):
    """The reference's own fp32 arithmetic (extract.py:148,191-194) on the GPU, TF32 off."""
    x = torch.nn.functional.normalize(f, p=2, dim=-1) if flags & NORMALIZE else f
    W = x @ x.transpose(1, 2)
    if flags & THRESHOLD:
        W = W * (W > 0)
    if not flags & NO_MAX:
        W = W / W.amax((1, 2), keepdim=True)
    return W


def check_real(f, flags, label, W=None, deg=None, counts=None, lam=0.0):
    """W (run here unless given) within _bound64 of float64; + lam counts rounds once more (u |W|)."""
    if W is None:
        W, deg = run_affinity(f, flags, counts, lam)
    N = f.shape[1]
    W64, Wb = _bound64(f, flags)
    ref = _fp32_reference(f, flags)
    if counts is not None:
        W64 = W64 + lam * counts.double()
        Wb = Wb * (1 + U) + U * W64.abs()
        ref = ref + float(lam) * counts.float()
    err = (W[:, :, :N].double() - W64).abs()
    ref_err = (ref.double() - W64).abs()
    scale = W64.abs().amax()
    print(f"\n{label}: kernel max|W - W64| {err.max():.3e} (bound {Wb.max():.3e}, {(err / Wb).max():.2f} of it), "
          f"fp32 reference {ref_err.max():.3e}; max|W64| {scale:.3e}")
    assert bool((err <= Wb).all()), f"{label}: {(err / Wb).max():.2f} x bound, {_diff(err > Wb)}"
    if deg is not None:
        derr = (deg.double() - W64.sum(2)).abs()
        dbound = Wb.sum(2) + N * U * W64.abs().sum(2) * (1 + 1e-3)
        assert bool((derr <= dbound).all()), f"{label}: degree {(derr / dbound).max():.2f} x bound"
    return err.max().item(), ref_err.max().item()


def _dino_features(dev, n):
    from oracle import dino_vit
    synth = load_pkg("synth")
    ref = dino_vit.build("dino_vits16", seed=0).to(dev)
    x = torch.cat([dino_vit.preprocess_u8(synth.blobs_image(480, 480, s), 16) for s in range(n)]).to(dev)
    return ref.forward_k(x).float().contiguous()


def _real_case(case, dev):
    synth = load_pkg("synth")
    g = torch.Generator(device="cpu").manual_seed(7)
    if case == "structured_196":
        return synth.structured_features(196, 384, 6, 196)[None].to(dev), NORMALIZE | THRESHOLD
    if case == "structured_900_b2":
        return torch.stack([synth.structured_features(900, 384, 6, s) for s in (1, 2)]).to(dev), NORMALIZE | THRESHOLD
    if case == "gauss_713_768":
        return torch.randn(1, 713, 768, generator=g).to(dev), NORMALIZE | THRESHOLD
    if case == "gauss_385_100_nothr":
        return torch.randn(1, 385, 100, generator=g).to(dev), NORMALIZE
    if case == "gauss_raw_300_64":
        return torch.randn(1, 300, 64, generator=g).to(dev), THRESHOLD
    if case == "dino_k_480":
        return _dino_features(dev, 2), NORMALIZE | THRESHOLD
    if case.startswith("spread"):   # row norms spread over 1e-3 .. 1e3
        x = torch.nn.functional.normalize(torch.randn(1, 500, 384, generator=g), dim=-1)
        x = x * 10.0 ** (6 * torch.rand(1, 500, 1, generator=g) - 3)
        return x.to(dev), NO_MAX | (THRESHOLD if case.endswith("thr") else 0)
    raise ValueError(case)


REAL_CASES = ["structured_196", "structured_900_b2", "gauss_713_768", "gauss_385_100_nothr", "gauss_raw_300_64",
              "dino_k_480", "spread_nomax", "spread_nomax_thr"]


@pytest.mark.parametrize("case", REAL_CASES)
def test_real_features_against_float64(cuda, case):
    f, flags = _real_case(case, cuda)
    check_real(f, flags, case)


# ---------------------------------------------------------------------------------------------------------------
# 4. batch independence at the benchmark's size
def test_batch_of_264_images_equals_each_image_alone(cuda):
    synth = load_pkg("synth")
    B, N, d = 264, 900, 384
    f = torch.stack([synth.structured_features(N, d, 6, 1000 + s) for s in range(B)]).to(cuda)
    W, deg = run_affinity(f, NORMALIZE | THRESHOLD)
    for z in range(B):
        W1, deg1 = run_affinity(f[z:z + 1], NORMALIZE | THRESHOLD)
        assert torch.equal(W[z], W1[0]) and torch.equal(deg[z], deg1[0]), f"image {z} differs from its run alone"
    for z in np.linspace(0, B - 1, 8).round().astype(int).tolist():
        check_real(f[z:z + 1], NORMALIZE | THRESHOLD, f"batch 264, image {z}", W[z:z + 1], deg[z:z + 1])


# ---------------------------------------------------------------------------------------------------------------
# 5. any row pitch ldw >= N, ldw % 4 == 0
@pytest.mark.parametrize("N,B", [(900, 2), (200, 3), (65, 1)])
def test_row_pitch(cuda, N, B):
    synth = load_pkg("synth")
    f = torch.stack([synth.structured_features(N, 384, 6, N + s) for s in range(B)]).to(cuda)
    c = _sym_counts(B, N, N, cuda)
    base = None
    for ldw in (_pitch(N), _roundup128(N), _roundup128(N) + 4, _roundup128(N) + 128):
        W, deg = run_affinity(f, NORMALIZE | THRESHOLD, c, 10.0, ldw=ldw)
        if base is None:
            base = (W, deg)
            check_real(f, NORMALIZE | THRESHOLD, f"ldw {ldw}", W, deg, c, 10.0)
        else:
            assert torch.equal(W[:, :, :N], base[0][:, :, :N]), f"ldw {ldw}: W differs from ldw {_pitch(N)}"
            assert torch.equal(deg, base[1]), f"ldw {ldw}: degree differs from ldw {_pitch(N)}"
    _check_degree_vs_W(deg, W, N)


# ---------------------------------------------------------------------------------------------------------------
# 6. colour terms
def _rgb_image(H, W, kind, seed):
    synth = load_pkg("synth")
    if kind == "blobs":
        return synth.blobs_image(H, W, seed).float().div(255.0)
    if kind == "uniform":
        return torch.full((H, W, 3), 0.4)
    if kind == "two_level":
        img = torch.full((H, W, 3), 0.2)
        img[:, W // 2:] = torch.tensor([0.7, 0.1, 0.5])
        return img
    raise ValueError(kind)


def _knn_counts(rgb, H, W):
    _l, lib = _lib()
    B, N = rgb.shape[0], H * W
    buf = torch.full(((B * N * N + 3) // 4 * 4 + 4096,), 0xEE, dtype=torch.uint8, device=rgb.device)
    _l.check(lib.dss_knn_color_counts(rgb.contiguous().data_ptr(), B, H, W, buf.data_ptr(), None, 0, _l.stream_ptr()),
             "dss_knn_color_counts")
    torch.cuda.synchronize()
    assert bool((buf[(B * N * N + 3) // 4 * 4:] == 0xEE).all()), "knn counts written past the buffer"
    return buf[:B * N * N].view(B, N, N)


def _knn_gpu(data, query, k):
    """eigs_ref.knn_exact on the GPU: fp32 squared distances accumulated dimension by dimension, (d2, index) order."""
    x = torch.from_numpy(np.ascontiguousarray(data)).cuda()
    d2 = torch.zeros(x.shape[0], x.shape[0], device="cuda")
    for c in range(x.shape[1]):
        diff = x[:, c:c + 1] - x[None, :, c]
        d2 += diff * diff
    _, idx = torch.sort(d2, dim=1, stable=True)
    return None, idx[:, :k].cpu().numpy()


@pytest.mark.parametrize("H,W,kind,B", [(4, 5, "blobs", 1), (1, 20, "blobs", 1), (20, 1, "blobs", 1),
                                        (12, 15, "uniform", 1), (9, 11, "two_level", 1), (80, 80, "blobs", 1),
                                        (5, 5, "blobs", 2), (7, 9, "blobs", 2), (64, 160, "blobs", 1)])
def test_knn_counts_match_oracle(cuda, H, W, kind, B):
    from oracle import eigs_ref
    imgs = [_rgb_image(H, W, kind, 31 * s + H) for s in range(B)]
    got = _knn_counts(torch.stack([im.reshape(-1, 3) for im in imgs]).to(cuda), H, W).cpu().numpy()
    knn = eigs_ref.knn_exact
    if H * W > 6400:   # the shared-memory maximum (5 N 4 bytes = 200 KB): the oracle's KNN restated on the GPU
        small = _rgb_image(30, 30, "blobs", 5).numpy().reshape(-1, 3)
        assert np.array_equal(_knn_gpu(small, small, 20)[1], eigs_ref.knn_exact(small, small, 20)[1])
        knn = _knn_gpu
    for b, im in enumerate(imgs):
        delta = eigs_ref.knn_affinity(im.numpy(), knn=knn) - scipy.sparse.csr_matrix(got[b]).astype(np.float64)
        delta.eliminate_zeros()
        assert delta.nnz == 0, f"image {b}: {delta.nnz} counts differ"


def test_knn_rejects_bad_sizes(cuda):
    _l, lib = _lib()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device=cuda)
    n0 = lib.dss_kernel_launch_count()
    assert lib.dss_knn_color_counts(buf.data_ptr(), 1, 1, 19, buf.data_ptr(), None, 0, _l.stream_ptr()) != 0
    assert lib.dss_knn_color_counts(buf.data_ptr(), 1, 1, 10241, buf.data_ptr(), None, 0, _l.stream_ptr()) != 0
    assert lib.dss_kernel_launch_count() == n0


@pytest.mark.parametrize("lam", [1.0, 10.0, 0.1])
def test_fused_knn_counts(cuda, lam):
    synth = load_pkg("synth")
    H = W_ = 14
    N = H * W_
    rgb = torch.stack([_rgb_image(H, W_, "blobs", s).reshape(-1, 3) for s in (3, 4)]).to(cuda)
    c = _knn_counts(rgb, H, W_)
    f = torch.stack([synth.structured_features(N, 384, 6, s) for s in (3, 4)]).to(cuda)
    W0, _ = run_affinity(f, NORMALIZE | THRESHOLD)
    W1, deg = run_affinity(f, NORMALIZE | THRESHOLD, c, lam)
    lam32 = torch.tensor(lam, dtype=torch.float32)
    want = (W0[:, :, :N].double() + (c.float() * lam32.to(cuda)).double()).float()
    if lam in (1.0, 10.0):
        assert torch.equal(W1[:, :, :N], want), _diff(W1[:, :, :N] != want)
    else:
        # the kernel's x += cnt * lambda contracts to one FMA (one rounding); the reference rounds cnt * lambda first
        ulp = (torch.nextafter(want.abs(), torch.tensor(float("inf"), device=cuda)) - want.abs())
        assert bool(((W1[:, :, :N] - want).abs() <= ulp).all())
    _check_degree_vs_W(deg, W1, N)


@pytest.mark.parametrize("H,W,B,ldw", [(1, 1, 1, None), (1, 7, 1, None), (6, 1, 1, None), (2, 2, 1, None),
                                       (30, 30, 3, None), (5, 9, 2, 64)])
def test_rw_affinity_add_matches_oracle(cuda, H, W, B, ldw):
    from oracle import eigs_ref
    _l, lib = _lib()
    N = H * W
    ldw = _pitch(N) if ldw is None else ldw
    g = torch.Generator().manual_seed(N)
    rgb = (128 + torch.randint(-6, 7, (B, N, 3), generator=g)).to(torch.uint8)
    if N >= 900:
        rgb = torch.stack([load_pkg("synth").blobs_image(H, W, s).reshape(-1, 3) for s in range(B)])
    lam = 3.0
    W0 = torch.full((B + 1, N, ldw), SENT)
    W0[:B, :, :N] = torch.rand(B, N, N, generator=g)
    deg0 = torch.cat([torch.rand(B, N, generator=g) * N, torch.full((1, N), SENT)])
    Wd, degd = W0.to(cuda), deg0.to(cuda)
    rgb_d = rgb.contiguous().to(cuda)
    _l.check(lib.dss_rw_affinity_add(rgb_d.data_ptr(), B, H, W, lam, 900.0, Wd.data_ptr(), ldw,
                                     degd.data_ptr(), _l.stream_ptr()), "dss_rw_affinity_add")
    torch.cuda.synchronize()
    Wd, degd = Wd.cpu(), degd.cpu()
    assert torch.equal(Wd[B], W0[B]) and torch.equal(Wd[:, :, N:], W0[:, :, N:]) and torch.equal(degd[B], deg0[B])
    for b in range(B):
        dense = np.asarray(eigs_ref.rw_affinity(rgb[b].numpy().reshape(H, W, 3) / 255.0).todense())
        add = torch.from_numpy(dense.astype(np.float32) * np.float32(lam))
        want = W0[b, :, :N] + add
        got = Wd[b, :, :N]
        ulp = torch.nextafter(want.abs(), torch.tensor(float("inf"))) - want.abs()
        assert bool(((got - want).abs() <= ulp).all()), f"image {b}: {_diff((got - want).abs() > ulp)}"
        assert torch.equal(got[add == 0], W0[b, :, :N][add == 0])
        a64 = torch.from_numpy(dense).sum(1) * lam
        dbound = 12 * U * (deg0[b].double().abs() + a64)
        assert bool(((degd[b].double() - (deg0[b].double() + a64)).abs() <= dbound).all())
