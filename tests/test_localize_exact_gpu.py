"""-m gpu: object localization at its edges, through the C ABI, exactly against the oracle (oracle/localize_ref.py).

Connected components: the masks of localize_ref.cc_patterns (row-end and row-wrap traps, U, serpentine, checkerboards,
equal largest components, 4096 roots, all / none / half set) on grids from 1 x 1 to 128 x 128, 1 x 16384 and
16384 x 1, reach the shared union-find through each kernel: eigen-segmentation from a +-1 row (8-connected), LOST
from an integer A whose similar rows add up to +-k per cell (4-connected, the seed placed by the degrees), DINO-seg from
dyadic attention rows (4-connected, the reference's component rule).

LOST: integer A is exact in fp32 in any summation order, so boxes and seeds are compared bit for bit at N 1, 8193,
16383 and 16384 (212 992 bytes of shared memory), k_patches 1 ... N + 5, with degree ties, zeros in the seed's row, no
similar at all and NaN / 1e30 in the pad columns of ldw > N; 300 images of 14 x 14 each equal their solo run. With
real-valued A the kernel equals the oracle's sequential fp32 sum bit for bit, and the reference's torch.sum wherever
float64 decides the sign; the undecidable cells are counted and printed.

DINO-seg: dyadic rows put a cumulative mass exactly on fl32(0.4), equal values on both sides of it, runs of zeros;
random rows are checked against the exactly rounded normalising sum always, and against torch's float sum wherever the
two keep the same cells.

The padded im2col bit for bit (the cropping im2col's own value table, +0.0 pad), and the CLS attention row against
float64 with a bound from its roundings. Outputs sit in buffers longer than the batch whose sentinels must survive,
workspaces start as 0xFF bytes, and every error status comes with a zero box."""
import math

import numpy as np
import pytest
import torch

from conftest import load_pkg
from oracle import localize_ref as L
from test_vit_exact_gpu import _im2col_domain

pytestmark = pytest.mark.gpu

GUARD = 37
SENT = -1234567
GRIDS = [(1, 1), (1, 16384), (16384, 1), (2, 8192), (63, 63), (127, 129), (128, 128)]


def _lib():
    _l = load_pkg("_lib")
    return _l, _l.load()


def _guarded(B, dev, width=1):
    return torch.full(((B + GUARD) * width,), SENT, dtype=torch.int32, device=dev)


def _ws(nbytes, dev):
    return torch.full((max(int(nbytes), 1),), 0xFF, dtype=torch.uint8, device=dev)


def _read(B, boxes, status, seeds=None):
    """(boxes int64 [B, 4], status [B], seeds [B] or None) after checking the sentinels and zero boxes on errors."""
    torch.cuda.synchronize()
    for buf, w in ((boxes, 4), (status, 1)) + (((seeds, 1),) if seeds is not None else ()):
        assert (buf[B * w:] == SENT).all(), "a sentinel after the outputs changed"
    bx = boxes[:B * 4].view(B, 4).cpu().numpy().astype(np.int64)
    st = status[:B].cpu().numpy()
    assert not bx[st != 0].any(), "an error status came with a nonzero box"
    return bx, st, (seeds[:B].cpu().numpy() if seeds is not None else None)


def _eigseg(V, sizes):
    """dss_eigseg_boxes on rows V [B, N] (K = 1, which = 0)."""
    _l, lib = _lib()
    B, N = V.shape
    dims = torch.tensor(sizes, dtype=torch.int32).contiguous()
    boxes, status = _guarded(B, V.device, 4), _guarded(B, V.device)
    nb = lib.dss_eigseg_boxes_workspace_bytes(B)
    ws = _ws(nb, V.device)
    _l.check(lib.dss_eigseg_boxes(V.data_ptr(), B, 1, N, 0, dims.data_ptr(), boxes.data_ptr(), status.data_ptr(),
                                  ws.data_ptr(), nb, _l.stream_ptr()), "eigseg")
    return _read(B, boxes, status)[:2]


def _lost(A, B, N, ldw, grid, size, P, k):
    """dss_lost_boxes on A [B, N, ldw] (any tensor whose storage starts there)."""
    _l, lib = _lib()
    boxes, status, seeds = _guarded(B, A.device, 4), _guarded(B, A.device), _guarded(B, A.device)
    nb = lib.dss_lost_workspace_bytes(B, N)
    ws = _ws(nb, A.device)
    _l.check(lib.dss_lost_boxes(A.data_ptr(), B, N, ldw, grid[0], grid[1], size[0], size[1], P, k, boxes.data_ptr(),
                                seeds.data_ptr(), status.data_ptr(), ws.data_ptr(), nb, _l.stream_ptr()), "lost")
    return _read(B, boxes, status, seeds)


def _dinoseg(attn, grid, P, head):
    """dss_dinoseg_boxes on attn [B, heads, N] fp32."""
    _l, lib = _lib()
    B, heads, N = attn.shape
    boxes, status = _guarded(B, attn.device, 4), _guarded(B, attn.device)
    _l.check(lib.dss_dinoseg_boxes(attn.data_ptr(), B, heads, N, head, grid[0], grid[1], P, boxes.data_ptr(),
                                   status.data_ptr(), _l.stream_ptr()), "dinoseg")
    return _read(B, boxes, status)[:2]


# ------------------------------------------------------------------------------------------------ eigen-segmentation
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_eigseg_cc_patterns(cuda, grid):
    """A +-1 row gives any mask: every pattern in one batch, boxes against skimage's 8-connected labels (scipy here).
    all / none: the flip to the whole grid; half (2s = N) is not flipped, half + 1 is; row_ends would merge a row's two
    ends through a missing c < gw - 1 guard; twin is a tie the smaller root must win."""
    gh, gw = grid
    pats = L.cc_patterns(gh, gw)
    V = torch.from_numpy(np.stack([np.where(m.ravel(), 1.0, -1.0) for m in pats.values()]).astype(np.float32))
    sizes = [(gh * 8 + 7, gw * 8 + 1)] * len(pats)
    boxes, status = _eigseg(V.to(cuda), sizes)
    assert (status == 0).all()
    for i, (name, m) in enumerate(pats.items()):
        want = L.eigseg_box(V[i].numpy(), *sizes[i])
        assert np.array_equal(boxes[i], want), (grid, name, boxes[i], want)


# ------------------------------------------------------------------------------------------------ LOST
def _rows(A, N):
    return lambda idx: A[torch.as_tensor(np.asarray(idx), device=A.device)][:, :N].cpu().numpy()


def _fill_pattern_A(A, m, placed):
    """A [N, ldw] <- every row +1 on the mask, -1 off it (ties: the seed is the smallest masked index; the similars sum
    to +-|S|). placed: the last masked cell becomes the seed through the degrees -- every other row gains +1 in the
    first unmasked column d, which the seed's row holds at -(N + 10), so M[d] stays negative. Pad columns: NaN / 1e30."""
    N = m.size
    mt = torch.from_numpy(m.ravel()).to(A.device)
    pat = torch.where(mt, 1.0, -1.0)
    A[:, :N] = pat
    A[0::2, N:] = float("nan")
    A[1::2, N:] = 1e30
    s0 = None
    if placed and 0 < m.sum() < N:
        s0, d = int(np.flatnonzero(m)[-1]), int(np.flatnonzero(~m.ravel())[0])
        A[:, d] = 1.0
        A[s0, :N] = pat
        A[s0, d] = -(N + 10.0)
    return s0


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_lost_cc_patterns(cuda, grid):
    """Designed integer A: the kernel's mask is the pattern, and box, seed and status equal the oracle's. Cell 0 is off
    most masks, so counting the diagonal in the degree moves the seed there. row_wrap would join a row's last cell to
    the next row's first through a missing c > 0 guard."""
    gh, gw = grid
    N, ldw = gh * gw, gh * gw + 3
    A = torch.empty(N, ldw, device=cuda)
    size, P = (gh * 16 - 3, gw * 16), 16
    for name, m in L.cc_patterns(gh, gw).items():
        for placed in (False, True):
            s0 = _fill_pattern_A(A, m, placed)
            if placed and s0 is None:
                continue
            boxes, status, seeds = _lost(A, 1, N, ldw, grid, size, P, 100)
            seed, _, M = L.lost_expand(_rows(A, N), N, 100)
            want, wst = L.detect_box(M, seed, grid, size, P)
            assert np.array_equal(M > 0, m.ravel()) or not m.any(), (grid, name)      # the construction
            assert seed == (s0 if placed else (int(np.flatnonzero(m)[0]) if m.any() else 0))
            assert (seeds[0], status[0]) == (seed, wst) and np.array_equal(boxes[0], want), (grid, name, placed)
    del A
    torch.cuda.empty_cache()


@pytest.mark.parametrize("N,grid", [(1, (1, 1)), (8193, (3, 2731)), (16383, (127, 129)), (16384, (128, 128))])
def test_lost_integer_A_every_k(cuda, N, grid):
    """A with entries in -3 .. 3 (zeros included), ldw = N + 5 with NaN / 1e30 pad columns: seeds, boxes and status
    equal the oracle's for k_patches 1, 31, 32, 33, 100, N, N + 5 (the similar list compacted across warp chunks)."""
    ldw = N + 5
    g = torch.Generator(device=cuda).manual_seed(N)
    A = torch.randint(-3, 4, (N, ldw), generator=g, device=cuda, dtype=torch.int8).float()
    A[:, N:N + 2] = float("nan")
    A[:, N + 2:] = 1e30
    size = (grid[0] * 8, grid[1] * 8 - 1)
    for k in (1, 31, 32, 33, 100, N, N + 5):
        boxes, status, seeds = _lost(A, 1, N, ldw, grid, size, 8, k)
        seed, _, M = L.lost_expand(_rows(A, N), N, k)
        want, wst = L.detect_box(M, seed, grid, size, 8)
        assert (seeds[0], status[0]) == (seed, wst) and np.array_equal(boxes[0], want), (N, k)
    del A
    torch.cuda.empty_cache()


@pytest.mark.parametrize("grid", [(63, 63), (128, 128)])
def test_lost_zero_in_seed_row_is_not_similar(cuda, grid):
    """A[seed, z] = 0 for the last potential z, whose row holds N + 10 next to the seed's block: z is not similar (the
    test is > 0), so that cell stays out of the box. Also: a seed row without any positive entry (status 2, seed
    reported), with all-zero and all-negative A."""
    gh, gw = grid
    N, ldw = gh * gw, gh * gw + 1
    m = np.zeros((gh, gw), bool)
    m[10:21, 10:21] = True
    A = torch.empty(N, ldw, device=cuda)
    _fill_pattern_A(A, m, False)
    z, y = N - 1, 15 * gw + 21
    A[10 * gw + 10, z] = 0.0
    A[z, y] = N + 10.0
    for k in (100, N, N + 5):
        boxes, status, seeds = _lost(A, 1, N, ldw, grid, (gh * 8, gw * 8), 8, k)
        seed, _, M = L.lost_expand(_rows(A, N), N, k)
        want, wst = L.detect_box(M, seed, grid, (gh * 8, gw * 8), 8)
        assert wst == 0 and np.array_equal(want, [80, 80, 168, 168])
        assert (seeds[0], status[0]) == (seed, 0) and np.array_equal(boxes[0], want), k
    for fill in (0.0, -1.0):
        A.fill_(fill)
        boxes, status, seeds = _lost(A, 1, N, ldw, grid, (gh * 8, gw * 8), 8, N)
        assert (seeds[0], status[0]) == (0, 2)
    del A
    torch.cuda.empty_cache()


def test_lost_batch_300_equals_solo_and_oracle(cuda):
    """300 images of 14 x 14 (two waves of 1024-thread CTAs on 132 SMs): every image equals its solo run and the oracle."""
    B, N, ldw, grid = 300, 196, 199, (14, 14)
    g = torch.Generator(device=cuda).manual_seed(300)
    A = torch.randint(-3, 4, (B, N, ldw), generator=g, device=cuda).float()
    A[..., N:] = float("nan")
    for k in (33, 100):
        boxes, status, seeds = _lost(A, B, N, ldw, grid, (220, 221), 16, k)
        for b in range(B):
            ob, os_, ose = _lost(A[b], 1, N, ldw, grid, (220, 221), 16, k)
            assert np.array_equal(ob[0], boxes[b]) and os_[0] == status[b] and ose[0] == seeds[b], (k, b)
            seed, _, M = L.lost_expand(_rows(A[b], N), N, k)
            want, wst = L.detect_box(M, seed, grid, (220, 221), 16)
            assert (seeds[b], status[b]) == (seed, wst) and np.array_equal(boxes[b], want), (k, b)


@pytest.mark.parametrize("grid,d,B,ks", [((24, 32), 64, 8, (100, 768)), ((64, 64), 64, 2, (100, 4096)),
                                         ((128, 128), 384, 1, (100, 1000))])
def test_lost_real_valued_A_summation_order(cuda, grid, d, B, ks):
    """A = F F^T of Gaussian features: boxes equal the oracle's sequential fp32 sum bit for bit, and the mask of the
    reference's CPU torch.sum(A[similars, :], 0) equals the sequential one at every cell float64 decides
    (|M| > gamma_nsim sum|A_sj|). The undecidable cells are counted and printed."""
    gh, gw = grid
    N = gh * gw
    g = torch.Generator(device=cuda).manual_seed(N + d)
    size = (gh * 16, gw * 16 - 9)
    undecided = flipped = total = 0
    for b in range(B):
        f = torch.randn(N, d, generator=g, device=cuda)
        A = f @ f.T
        for k in ks:
            boxes, status, seeds = _lost(A, 1, N, N, grid, size, 16, k)
            seed, sim, M = L.lost_expand(_rows(A, N), N, k)
            want, wst = L.detect_box(M, seed, grid, size, 16)
            assert (seeds[0], status[0]) == (seed, wst) and np.array_equal(boxes[0], want), (b, k)
            rows = _rows(A, N)(sim)
            m64, decided = L.sum_decided(rows)
            mt = torch.sum(torch.from_numpy(rows), dim=0).numpy()
            differ = (M > 0) != (mt > 0)
            assert not differ[decided].any()
            undecided += int((~decided).sum())
            flipped += int(differ.sum())
            total += N
            if not differ.any():
                assert np.array_equal(L.detect_box(mt, seed, grid, size, 16)[0], boxes[0])
        del A, f
    torch.cuda.empty_cache()
    print(f"LOST {gh}x{gw}: {undecided} of {total} cells undecidable, {flipped} flipped by torch's summation order")


# ------------------------------------------------------------------------------------------------ DINO-seg
def _dyadic(m, tie_cell=None):
    return (L.dyadic_row(m, tie_cell) * L.DYADIC_UNIT).astype(np.float32)


def _attn(rows, heads, head):
    """[B, heads, N] with rows in `head` and the other heads holding other rows of the batch (a wrong head, a wrong box)."""
    rows = np.stack(rows)
    a = np.stack([np.roll(rows, h - head + 1, axis=0) if h != head else rows for h in range(heads)], 1)
    return torch.from_numpy(np.ascontiguousarray(a))


@pytest.mark.parametrize("heads", [6, 12])
@pytest.mark.parametrize("grid", GRIDS + [(8, 12)], ids=[f"{h}x{w}" for h, w in GRIDS + [(8, 12)]])
def test_dinoseg_dyadic_patterns(cuda, grid, heads):
    """Dyadic rows keep exactly the pattern's cells (a cumulative mass on fl32(0.4) itself is not kept): the reference's
    rule picks the largest of labels 1 .. n - 1, the background for n <= 1, nothing (status 3) when every cell is kept."""
    gh, gw = grid
    rows, names = [], []
    for name, m in L.cc_patterns(gh, gw).items():
        try:
            rows.append(_dyadic(m))
        except ValueError:
            continue
        names.append(name)
    assert len(names) >= (3 if gh * gw > 1 else 0)
    if gh * gw <= 2:
        return
    head = heads - 1
    boxes, status = _dinoseg(_attn(rows, heads, head).to(cuda), grid, 8, head)
    for i, name in enumerate(names):
        kept = L.dinoseg_kept(rows[i])
        assert np.array_equal(kept, L.cc_patterns(gh, gw)[name].ravel())
        want, wst = L.dinoseg_select(kept, grid, 8)
        assert status[i] == wst and np.array_equal(boxes[i], want), (grid, name)


def test_dinoseg_threshold_ties_and_empty_selection(cuda):
    """A non-kept cell above the winning block shares the lowest kept value; its index is smaller, so it sorts first and
    its cumulative mass is exactly fl32(0.4): not kept (> 0.4), and the block's first cell is. A last-numbered single
    cell makes n = 2, so the block wins. 1 x 1 and 1 x 2 grids keep every cell: status 3."""
    for gh, gw in [(8, 12), (63, 63), (128, 128)]:
        m = np.zeros((gh, gw), bool)
        m[3:6, 4:8] = True
        m[gh - 1, gw - 1] = True
        row = _dyadic(m, tie_cell=2 * gw + 4)
        for heads in (6, 12):
            boxes, status = _dinoseg(_attn([row, row[::-1].copy()], heads, heads - 1).to(cuda), (gh, gw), 16, heads - 1)
            assert status[0] == 0 and np.array_equal(boxes[0], [64, 48, 128, 96]), (gh, gw, boxes[0])
            want, wst = L.dinoseg_select(L.dinoseg_kept(row), (gh, gw), 16)
            assert np.array_equal(boxes[0], want) and wst == 0
            want, wst = L.dinoseg_select(L.dinoseg_kept(row[::-1].copy()), (gh, gw), 16)
            assert status[1] == wst and np.array_equal(boxes[1], want)
    for row, grid in [([1.0], (1, 1)), ([0.4375, 0.5625], (1, 2))]:
        boxes, status = _dinoseg(torch.tensor([[row] * 6], device=cuda), grid, 16, 5)
        assert status[0] == 3 and L.dinoseg_select(L.dinoseg_kept(np.float32(row)), grid, 16)[1] == 3


def test_dinoseg_batch_300_equals_solo_and_oracle(cuda):
    rng = np.random.default_rng(300)
    grid, N = (14, 14), 196
    rows = []
    while len(rows) < 300:
        try:
            rows.append(_dyadic(rng.random((14, 14)) < rng.uniform(0.05, 0.5)))
        except ValueError:
            pass
    a = _attn(rows, 6, 5).to(cuda)
    boxes, status = _dinoseg(a, grid, 16, 5)
    for b in range(300):
        ob, os_ = _dinoseg(a[b:b + 1].contiguous(), grid, 16, 5)
        assert np.array_equal(ob[0], boxes[b]) and os_[0] == status[b], b
        want, wst = L.dinoseg_select(L.dinoseg_kept(rows[b]), grid, 16)
        assert status[b] == wst and np.array_equal(boxes[b], want), b


@pytest.mark.parametrize("grid,spread", [((24, 32), 2.0), ((63, 63), 2.0), ((128, 128), 2.0), ((128, 128), 30.0)])
def test_dinoseg_random_rows_decision(cuda, grid, spread):
    """Softmax rows (a spread of 30 underflows most of a row to exact zeros): the kernel equals the oracle with the
    exactly rounded normalising sum always, and the oracle with torch's float sum wherever the two keep the same cells."""
    gh, gw = grid
    rng = np.random.default_rng(gh + int(spread))
    s = rng.normal(0, spread, (8, 6, gh * gw))
    a = np.exp(s - s.max(-1, keepdims=True))
    a = (a / a.sum(-1, keepdims=True)).astype(np.float32)
    boxes, status = _dinoseg(torch.from_numpy(a).to(cuda), grid, 16, 4)
    differ = 0
    for b in range(8):
        k64, kt = L.dinoseg_kept(a[b, 4], "fp64"), L.dinoseg_kept(a[b, 4])
        want, wst = L.dinoseg_select(k64, grid, 16)
        assert status[b] == wst and np.array_equal(boxes[b], want), b
        if np.array_equal(k64, kt):
            assert np.array_equal(boxes[b], L.dinoseg_select(kt, grid, 16)[0])
        else:
            differ += 1
    print(f"DINO-seg {gh}x{gw} spread {spread}: {differ} of 8 rows keep other cells under torch's float sum")


# ------------------------------------------------------------------------------------------------ ViT pieces
def _im2col_pad(img, P):
    _l, lib = _lib()
    B, H, W, _ = img.shape
    rows = B * -(-H // P) * -(-W // P)
    buf = torch.full((rows + GUARD, 3 * P * P), float("nan"), dtype=torch.float16, device=img.device)
    buf[rows:] = -777.5
    _l.check(lib.dss_op_im2col_pad_f16(img.data_ptr(), buf.data_ptr(), B, H, W, P, _l.stream_ptr()), "im2col_pad")
    torch.cuda.synchronize()
    assert (buf[rows:] == -777.5).all(), "sentinel rows after the output changed"
    return buf[:rows]


@pytest.mark.parametrize("P", [8, 16])
def test_im2col_pad_bit_for_bit(cuda, P):
    """Every element inside the image is the cropping im2col's own (byte, channel) value, every pad element +0.0
    bitwise: H and W at every remainder mod P (0 included), 8-pixel groups across the right edge, images smaller than
    a patch, B = 3."""
    lut = _im2col_domain(cuda)
    ch = torch.arange(3, device=cuda)
    shapes = [(2 * P + r, 3 * P + (5 * r + 3) % P) for r in range(P)] + [(P + 3, 2 * P + r) for r in range(P)]
    shapes += [(1, 1), (1, P + 1), (P - 1, 1)]
    g = torch.Generator(device=cuda).manual_seed(P)
    for H, W in shapes:
        img = torch.randint(0, 256, (3, H, W, 3), generator=g, device=cuda, dtype=torch.uint8)
        out = _im2col_pad(img, P)
        Hp, Wp = -(-H // P), -(-W // P)
        want = torch.zeros(3, Hp * P, Wp * P, 3, dtype=torch.float16, device=cuda)
        want[:, :H, :W] = lut[ch, img.long()]
        want = want.view(3, Hp, P, Wp, P, 3).permute(0, 1, 3, 5, 2, 4).reshape(3 * Hp * Wp, 3 * P * P)
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)), (H, W)


def _cls(qkv, heads):
    _l, lib = _lib()
    B, T, _ = qkv.shape
    n = B * heads * (T - 1)
    buf = torch.full((n + GUARD,), float("nan"), device=qkv.device)
    buf[n:] = -7777.25
    _l.check(lib.dss_op_cls_attention(qkv.data_ptr(), B, T, heads, buf.data_ptr(), _l.stream_ptr()), "cls_attention")
    torch.cuda.synchronize()
    assert (buf[n:] == -7777.25).all()
    return buf[:n].view(B, heads, T - 1)


@pytest.mark.parametrize("T", [2, 257, 901, 3601, 6401])
def test_cls_attention_float64_bound(cuda, T):
    """Per element against float64, within localize_ref.cls_attention_bound (derived from the kernel's roundings),
    logits of standard deviation 3. Equal scores give fl(1 / T) exactly; one dominating score (by 256) gives exactly 1
    there and exactly 0 elsewhere, also when it is the CLS token's own."""
    for heads in (6, 12):
        d = heads * 64
        g = torch.Generator(device=cuda).manual_seed(T + heads)
        qkv = (torch.randn(2, T, 3 * d, generator=g, device=cuda) * math.sqrt(3)).half()
        qkv[:, 1:, :d] = float("nan")            # q of the other tokens and all of v are never read
        qkv[:, :, 2 * d:] = float("nan")
        got = _cls(qkv, heads).double().cpu()
        p, bound = L.cls_attention_bound(qkv, heads)
        err = (got - p).abs()
        assert (err <= bound).all(), f"T={T} heads={heads}: worst err / bound {float((err / bound).max()):.3f}"
        # equal scores, and one score dominating by 256 (q = 4, k = 8: 64 * 32 / 8), at token 0 and at token T // 2
        for dom in (None, 0, T // 2):
            qkv[:, 0, :d] = 4.0
            qkv[:, :, d:2 * d] = 0.0 if dom is not None else 0.5
            if dom is not None:
                qkv[:, dom, d:2 * d] = 8.0
            got = _cls(qkv, heads).cpu()
            want = torch.full_like(got, np.float32(1.0 / T) if dom is None else 0.0)
            if dom:
                want[..., dom - 1] = 1.0
            assert torch.equal(got, want), (T, heads, dom)
