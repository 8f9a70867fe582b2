"""-m gpu: the ViT forward's own kernels checked exactly, or against float64 with a bound derived from where they round.

GEMM (dss_op_gemm_f16, dss_debug_gemm_cfg): A and Wt hold small integers stored as fp16, the bias is integer-valued and
the positional embedding a multiple of 2^-8. Every product is then exact and every partial sum an integer below 2^20,
so an fp32 sum of them is exact in any order: the float64 product is THE answer and outputs are compared with
torch.equal (fp16 outputs against the float64 value rounded once to fp16, overflow to inf included). The GELU
epilogue must lie within half an fp16 ulp plus the approximation's 6.4e-6 of the float64 GELU of the exact
accumulator (compared unrounded: its fp16 rounding may fall on the other side of a midpoint). The shapes reach
all six epilogues, all three tile widths, partial n-tiles, ring depths below / equal to / not dividing the number of
K slabs, and the benchmark's 264-image row counts, where every CTA pair runs many tiles in a row.

Attention (dss_op_attention_tc_f16): float64 softmax of the same fp16 qkv; the per-element bound follows the kernel's
roundings (P to fp16, fp32 scores and sums, fp16 output), not the largest element. Every image of a batch must be
bitwise equal to the same image run alone, also at the benchmark's batch through the whole ViT.

im2col over its complete input domain (256 byte values x 3 channels), LayerNorm against float64 with a bound that
holds for a two-pass variance only.

Every output buffer is NaN-filled and followed by GUARD sentinel rows that must stay untouched."""
import math

import numpy as np
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

GUARD = 128
SENT = {torch.float32: -7777.25, torch.float16: -777.5}
EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RESID_F32, EPI_BIAS_F32, EPI_PATCH_F32, EPI_DROPCLS_F32 = range(6)
EPI_NAME = {EPI_BIAS_F16: "f16", EPI_BIAS_GELU_F16: "gelu", EPI_BIAS_RESID_F32: "resid", EPI_BIAS_F32: "f32",
            EPI_PATCH_F32: "patch", EPI_DROPCLS_F32: "dropcls"}
GELU_ERR = 6.5e-6   # max |gelu_erf - gelu| over the fp32 range is 6.4e-6 (csrc/common.cuh)


def _lib():
    _l = load_pkg("_lib")
    return _l, _l.load()


def _ulp16(a):
    """Spacing of fp16 at |a| (float64 tensor): 2^(e - 10) in the normal range, 2^-24 below it."""
    return torch.exp2(torch.floor(torch.log2(a.abs().clamp(min=2.0 ** -14))) - 10)


def _out_buffer(rows, cols, dtype, dev):
    buf = torch.full((rows + GUARD, cols), float("nan"), dtype=dtype, device=dev)
    buf[rows:] = SENT[dtype]
    return buf


def _assert_guard(buf, rows):
    assert torch.equal(buf[rows:], torch.full_like(buf[rows:], SENT[buf.dtype])), "sentinel rows after the output changed"


def _diff(bad, r0=0):
    idx = bad.nonzero()[:6].tolist()
    return f"{int(bad.sum())} of {bad.numel()} elements differ, first at (row, col) {[(r + r0, c) for r, c in idx]}"


# ---------------------------------------------------------------------------------------------------------------
# GEMM, bit for bit
def _gemm_operands(epi, M, N, K, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    A = torch.randint(-4, 5, (M, K), generator=g, device=dev, dtype=torch.int8)
    Wt = torch.randint(-4, 5, (N, K), generator=g, device=dev, dtype=torch.int8).half()
    if epi == EPI_BIAS_GELU_F16:
        # accumulators: multiples of 2^-6 that densely cover [-10, 10] (row scales 1..3 widen the spread)
        A = A * torch.randint(1, 4, (M, 1), generator=g, device=dev, dtype=torch.int8)
        Wt = Wt * 2.0 ** -6
        bias = torch.randint(-128, 129, (N,), generator=g, device=dev).float() * 2.0 ** -6
    else:
        bias = torch.randint(-8, 9, (N,), generator=g, device=dev).float()
    A = A.half()
    if epi != EPI_PATCH_F32 and epi != EPI_BIAS_GELU_F16:
        # hot rows / columns: accumulators above 2048 (fp16 round-to-even) and above 65504 (fp16 overflow to inf);
        # the largest partial sum, 64 * 4 * 1536, stays below 2^20
        A[::97] = 64.0
        Wt[::29] = 4.0
        Wt[1::29] = -4.0
    return A, Wt, bias


def _gemm_case(dev, epi, M, N, K, seed, rin=0, rout=0, bn=None):
    """Runs one GEMM into a NaN-filled, guarded buffer and checks it against the exact float64 product."""
    _l, lib = _lib()
    A, Wt, bias = _gemm_operands(epi, M, N, K, seed, dev)
    g = torch.Generator(device=dev).manual_seed(seed + 1)
    out16 = epi in (EPI_BIAS_F16, EPI_BIAS_GELU_F16)
    rows = M // rin * rout if epi in (EPI_PATCH_F32, EPI_DROPCLS_F32) else M
    buf = _out_buffer(rows, N, torch.float16 if out16 else torch.float32, dev)
    aux = x0 = None
    if epi == EPI_PATCH_F32:
        aux = torch.randint(-2048, 2049, (rout, N), generator=g, device=dev).float() * 2.0 ** -8
    if epi == EPI_BIAS_RESID_F32:
        x0 = torch.randint(-1024, 1025, (M, N), generator=g, device=dev).float()
        buf[:M] = x0
    st = _l.stream_ptr()
    if bn is None:
        _l.check(lib.dss_op_gemm_f16(A.data_ptr(), Wt.data_ptr(), bias.data_ptr(), buf.data_ptr(), M, N, K, epi,
                                     None if aux is None else aux.data_ptr(), rin, rout, st), "gemm")
    else:
        assert epi == EPI_BIAS_F16
        _l.check(lib.dss_debug_gemm_cfg(A.data_ptr(), Wt.data_ptr(), bias.data_ptr(), buf.data_ptr(), M, N, K, bn, 0, st),
                 "gemm_cfg")
    torch.cuda.synchronize()
    _assert_guard(buf, rows)

    Wt64, b64 = Wt.double().T.contiguous(), bias.double()
    chunk = max(128, (1 << 24) // N)
    worst_gelu, flips = 0.0, 0
    for r0 in range(0, M, chunk):
        r1 = min(M, r0 + chunk)
        ref = torch.addmm(b64, A[r0:r1].double(), Wt64)   # exact: integers (multiples of 2^-6) far below 2^53
        m = torch.arange(r0, r1, device=dev)
        if epi == EPI_PATCH_F32:
            t = m % rin
            ref += aux.double()[t + 1]
            got = buf[(m // rin) * rout + t + 1]
        elif epi == EPI_DROPCLS_F32:
            t = m % rin
            keep = t != 0
            ref = ref[keep]
            got = buf[((m // rin) * rout + t - 1)[keep]]
        else:
            if epi == EPI_BIAS_RESID_F32:
                ref += x0[r0:r1].double()
            got = buf[r0:r1]
        if epi == EPI_BIAS_GELU_F16:
            gelu = ref * 0.5 * (1.0 + torch.erf(ref * (0.5 ** 0.5)))
            g64 = got.double()
            err = (g64 - gelu).abs()
            bound = 0.5 * _ulp16(torch.maximum(gelu.abs(), g64.abs())) + GELU_ERR
            bad = ~(err <= bound)
            assert not bad.any(), f"GELU epilogue beyond 0.5 ulp16 + {GELU_ERR}: {_diff(bad, r0)}"
            # the share of the approximation allowance used beyond the fp16 rounding
            worst_gelu = max(worst_gelu, float(((err - (bound - GELU_ERR)) / GELU_ERR).max()))
            flips += int((got != gelu.float().half()).sum())
        else:
            want = ref.half() if out16 else ref.float()   # ref is an integer below 2^24: one rounding to fp16
            if not torch.equal(got, want):
                bad = got != want
                raise AssertionError(f"{EPI_NAME[epi]} M={M} N={N} K={K} bn={bn}: {_diff(bad, r0)}; "
                                     f"got {got[bad][:4].tolist()} want {want[bad][:4].tolist()}")
    if epi == EPI_PATCH_F32:   # the CLS row of every image keeps its NaN
        assert torch.isnan(buf[torch.arange(M // rin, device=dev) * rout]).all(), "PATCH epilogue wrote a CLS row"
    if epi == EPI_BIAS_GELU_F16:
        print(f"gelu M={M} N={N} K={K}: worst (err - 0.5 ulp16) / {GELU_ERR} = {worst_gelu:.3f}, "
              f"{flips} outputs one fp16 ulp from fp16(gelu64)")
    return buf


TILE_N = [1536, 2304, 1152, 384, 640, 160, 96]   # tile widths 256, 256, 192, 192, 128, 128 (partial), 128 (partial)


@pytest.mark.parametrize("N", TILE_N)
@pytest.mark.parametrize("epi", [EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_F32, EPI_BIAS_RESID_F32],
                         ids=lambda e: EPI_NAME[e])
def test_gemm_exact_tile_widths(cuda, epi, N):
    # 8 images of 901 rows: 29 row pairs x up to 9 n-tiles, more work items than clusters
    _gemm_case(cuda, epi, 8 * 901, N, 384, seed=N + 17 * epi)


@pytest.mark.parametrize("N", [640, 384], ids=["bn128_6stages", "bn192_4stages"])
@pytest.mark.parametrize("K", [8, 72, 192, 256, 384, 768, 1536])
def test_gemm_exact_k_slabs(cuda, K, N):
    # num_kb = 1, 2 (zero-filled tail slab), 3, 4, 6, 12, 24 against rings of 6 (BN 128) and 4 (BN 192) stages
    _gemm_case(cuda, EPI_BIAS_F16, 8 * 901, N, K, seed=K + N)


def _remap(epi, M):
    if epi == EPI_PATCH_F32:
        rin = 900 if M % 900 == 0 else M
        return rin, rin + 1
    if epi == EPI_DROPCLS_F32:
        rin = 901 if M % 901 == 0 else M
        return rin, rin - 1
    return 0, 0


ROW_CASES = [(epi, M) for epi in EPI_NAME for M in (128, 129, 3 * (900 if epi == EPI_PATCH_F32 else 901))]


@pytest.mark.parametrize("epi,M", ROW_CASES, ids=[f"{EPI_NAME[e]}-M{m}" for e, m in ROW_CASES])
def test_gemm_exact_rows(cuda, epi, M):
    # M = 128: the odd CTA's tile lies wholly out of bounds; 129: one live row in it; 3 images of 900 / 901 rows
    rin, rout = _remap(epi, M)
    _gemm_case(cuda, epi, M, 384, 768 if epi == EPI_PATCH_F32 else 384, seed=M + epi, rin=rin, rout=rout)


def test_gemm_forced_tile_widths_agree(cuda):
    outs = [_gemm_case(cuda, EPI_BIAS_F16, 8 * 901, 768, 384, seed=5, bn=bn) for bn in (128, 192, 256)]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


BENCH_B = 264   # images per step of the benchmark (2 x 132 SMs)


BENCH_GEMMS = [   # the ViT-S/16 GEMMs of one benchmark step (480^2: 900 patches, 901 tokens per image)
    ("qkv", EPI_BIAS_F16, BENCH_B * 901, 1152, 384, 0, 0),
    ("proj", EPI_BIAS_RESID_F32, BENCH_B * 901, 384, 384, 0, 0),
    ("fc1", EPI_BIAS_GELU_F16, BENCH_B * 901, 1536, 384, 0, 0),
    ("fc2", EPI_BIAS_RESID_F32, BENCH_B * 901, 384, 1536, 0, 0),
    ("patch", EPI_PATCH_F32, BENCH_B * 900, 384, 768, 900, 901),
    ("kproj", EPI_DROPCLS_F32, BENCH_B * 901, 384, 384, 901, 900),
]


@pytest.mark.parametrize("name,epi,M,N,K,rin,rout", BENCH_GEMMS, ids=[c[0] for c in BENCH_GEMMS])
def test_gemm_exact_bench_shapes(cuda, name, epi, M, N, K, rin, rout):
    torch.cuda.reset_peak_memory_stats()
    _gemm_case(cuda, epi, M, N, K, seed=len(name) * 1000 + epi, rin=rin, rout=rout)
    print(f"{name}: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# Attention against float64
ATT_B = 5
ATT_SAFETY = 1.25   # on the modelled fp32 / fp16 rounding terms below (all of them upper bounds already)


def _att_qkv(B, T, heads, seed, dev):
    """fp16 qkv [B*T, 3*64*heads]. Odd images: K scaled by 30 and V = +-60000, so an even image that reads the next
    image's keys past T (the last key tile is partial) would show a gross error. In every image: row 0 has q = 0 (all
    scores equal), row 1 one dominant key (key 0, score 40 above the rest), rows 2 and 3 their maximum at key T-1 (the
    last key tile) and T//2 (score 12)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    shape = (B, T, heads, 64)
    q = torch.randn(shape, generator=g, device=dev) * 1.5
    k = torch.randn(shape, generator=g, device=dev) * 1.5
    v = torch.randn(shape, generator=g, device=dev) * 1.5
    odd = torch.arange(B, device=dev) % 2 == 1
    k[odd] *= 30.0
    sign = torch.randint(0, 2, shape, generator=g, device=dev).float() * 2 - 1
    v[odd] = sign[odd] * 60000.0
    k16 = k.half().float()

    def aim(row, key, score):
        if row < T:
            kr = k16[:, key]
            q[:, row] = kr * (8.0 * score / (kr * kr).sum(-1, keepdim=True))

    q[:, 0] = 0.0
    aim(1, 0, 40.0)
    aim(2, T - 1, 12.0)
    aim(3, T // 2, 12.0)
    return torch.stack([q, k, v], dim=2).reshape(B * T, 3 * heads * 64).half()


def _att_run(qkv, B, T, heads):
    _l, lib = _lib()
    buf = _out_buffer(B * T, heads * 64, torch.float16, qkv.device)
    _l.check(lib.dss_op_attention_tc_f16(qkv.data_ptr(), buf.data_ptr(), B, T, heads, _l.stream_ptr()), "attention")
    torch.cuda.synchronize()
    _assert_guard(buf, B * T)
    return buf[:B * T]


def _att_ref_and_bound(qkv, B, T, heads):
    """float64 O = softmax(Q K^T / 8) V and a per-element bound on |O_kernel - O| from the kernel's roundings:
      - scores: 64-term fp32 dot products summed 16 products per k-step over 4 k-steps, error <= 8 2^-23 sum|q k|
        (depth of the sum, each step rounded or truncated); relative p error: that / 8, for the key and for the row
        maximum;
      - p = ex2.approx(s c - m c): 2 ulp plus the fp32 rounding of m c (2^-23 |m| relative);
      - P rounded to fp16 for the PV product: relative 2^-11 (normal), absolute 2^-25 (subnormal);
      - the row sum l is taken over the unrounded p, in fp32 (relative T 2^-24); PV accumulates in fp32 over
        ceil(T / 16) k-steps plus one rescale per key tile;
      - O = (PV) * (1 / l), then rounded to fp16: half an fp16 ulp of the result."""
    x = qkv.double().view(B, T, 3, heads, 64).permute(2, 0, 3, 1, 4)   # [3, B, H, T, 64]
    q, k, v = x[0], x[1], x[2]
    S = q @ k.transpose(-1, -2) / 8
    m = S.amax(-1, keepdim=True)
    p = torch.exp(S - m)
    del S
    l = p.sum(-1, keepdim=True)
    o = (p @ v) / l
    pv = p @ v.abs()
    del p
    dot_err = (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True) * 8 * 2.0 ** -23
    e_p = dot_err / 4 + 2.0 ** -21 + 2.0 ** -23 * m.abs()
    e_num = 2.0 ** -11 + e_p + (math.ceil(T / 16) + 16) * 2.0 ** -23
    e_l = T * 2.0 ** -24 + e_p + 2.0 ** -22
    pre = ATT_SAFETY * ((e_num * pv + 2.0 ** -25 * v.abs().sum(-2, keepdim=True)) / l + o.abs() * e_l)
    bound = pre + 0.5 * _ulp16(o.abs() + pre)
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * T, heads * 64)
    return flat(o), flat(bound)


@pytest.mark.parametrize("heads", [6, 12])
@pytest.mark.parametrize("T", [1, 2, 4, 17, 63, 64, 65, 127, 128, 129, 255, 257, 901])
def test_attention_float64_bound_and_batch_independence(cuda, T, heads):
    qkv = _att_qkv(ATT_B, T, heads, seed=T * 31 + heads, dev=cuda)
    out = _att_run(qkv, ATT_B, T, heads)
    o, bound = _att_ref_and_bound(qkv, ATT_B, T, heads)
    err = (out.double() - o).abs()
    ok = err <= bound          # NaN fails
    ratio = err / bound
    worst = float(ratio.max())
    print(f"attention T={T} heads={heads}: worst err/bound {worst:.3f} (margin {1 - worst:.3f}), "
          f"max err {float(err.max()):.3e}")
    assert ok.all(), f"attention beyond its rounding bound: {_diff(~ok)}; worst err/bound {worst:.2f}"
    # no coupling between the images of a batch: each one alone gives the same bits
    for b in range(ATT_B):
        alone = _att_run(qkv[b * T:(b + 1) * T].contiguous(), 1, T, heads)
        assert torch.equal(alone, out[b * T:(b + 1) * T]), f"image {b} differs when run alone"


# ---------------------------------------------------------------------------------------------------------------
# The benchmark's batch through the whole ViT, bitwise against single images
@pytest.fixture(scope="module")
def vit_pair(cuda):
    from oracle import dino_vit
    vit = load_pkg("vit")
    ref = dino_vit.build("dino_vits16", seed=0)
    mine = vit.DinoViT("dino_vits16", ref.state_dict(), device=cuda)
    return ref.to(cuda), mine


def test_forward_k_bench_batch_equals_single_images(cuda, vit_pair):
    synth = load_pkg("synth")
    _, mine = vit_pair
    imgs = synth.blobs_batch(BENCH_B, 480, 480, seed0=0).to(cuda)
    torch.cuda.reset_peak_memory_stats()
    k = mine.forward_k(imgs)
    torch.cuda.synchronize()
    assert torch.isfinite(k).all()
    for i in (0, 1, 65, 66, 131, 132, BENCH_B - 1):
        k1 = mine.forward_k(imgs[i:i + 1])
        assert torch.equal(k1[0], k[i]), f"image {i} of the {BENCH_B}-image batch differs from the image alone"
    print(f"forward_k {BENCH_B} x 480^2: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    mine._ws = None
    del k, imgs
    torch.cuda.empty_cache()


@pytest.mark.parametrize("H,W", [(16, 16), (16, 48)])
def test_forward_cls_crop_batch_equals_single_crops(cuda, vit_pair, H, W):
    """Bounding-box crops of one and three patches (T = 2, 4): batch of 32 vs each crop alone, and the fp32 oracle."""
    from oracle import dino_vit
    synth = load_pkg("synth")
    ref, mine = vit_pair
    imgs = synth.blobs_batch(32, H, W, seed0=100 + W)
    got = mine.forward_cls(imgs.to(cuda)).clone()
    for i in range(imgs.shape[0]):
        one = mine.forward_cls(imgs[i:i + 1].to(cuda))
        assert torch.equal(one[0], got[i]), f"crop {i} of the batch differs from the crop alone"
    want = ref(torch.cat([dino_vit.preprocess_u8(im, 16) for im in imgs]).to(cuda))
    rel = float((got - want).norm() / want.norm())
    print(f"CLS {H}x{W} x 32: rel-L2 vs fp32 oracle {rel:.3e}")
    assert rel <= 3e-3


# ---------------------------------------------------------------------------------------------------------------
# im2col over its whole input domain; LayerNorm against float64
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def _im2col(img, P):
    _l, lib = _lib()
    B, H, W, _ = img.shape
    rows = B * (H // P) * (W // P)
    buf = _out_buffer(rows, 3 * P * P, torch.float16, img.device)
    _l.check(lib.dss_op_im2col_f16(img.data_ptr(), buf.data_ptr(), B, H, W, P, _l.stream_ptr()), "im2col")
    torch.cuda.synchronize()
    _assert_guard(buf, rows)
    return buf[:rows]


def _im2col_domain(dev):
    """The kernel's fp16 value of every (byte, channel) pair as a [3, 256] table, from one 16 x 256 image whose column x
    holds byte (x + 85 c) % 256 in channel c (so each channel sees all 256 values, at 16 rows each)."""
    P, H, W = 16, 16, 256
    x = torch.arange(W)
    img = torch.stack([((x + 85 * c) % 256)[None, :].expand(H, W) for c in range(3)], -1).to(torch.uint8)
    out = _im2col(img[None].to(dev), P)                                   # [16 patches, 3*16*16]
    pix = out.view(W // P, 3, P, P).permute(2, 0, 3, 1).reshape(H, W, 3)  # back to [y, x, c]
    assert torch.equal(pix, pix[:1].expand(H, W, 3)), "im2col: equal pixels of one column came out different"
    lut = torch.empty(3, 256, dtype=torch.float16, device=dev)
    for c in range(3):
        lut[c, img[0, :, c].long().to(dev)] = pix[0, :, c]
    return lut


def test_im2col_whole_input_domain(cuda):
    lut = _im2col_domain(cuda).cpu()
    u = np.arange(256, dtype=np.float64)
    want = np.stack([((u / 255.0 - MEAN[c]) / STD[c]).astype(np.float16) for c in range(3)])   # one rounding
    got = lut.numpy()
    ulp = _ulp16(torch.from_numpy(np.maximum(np.abs(want), np.abs(got)).astype(np.float64))).numpy()
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    inexact = int((got != want).sum())
    print(f"im2col: {inexact} of 768 (byte, channel) inputs are not the correctly rounded fp16 value")
    assert (err <= ulp).all(), np.argwhere(err > ulp)[:8]


@pytest.mark.parametrize("B,H,W,P", [(BENCH_B, 480, 480, 16), (3, 61, 75, 8)])
def test_im2col_layout(cuda, B, H, W, P):
    """Every patch element is the kernel's own table value of its (byte, channel) at the right place. 61 x 75 at P = 8:
    the crop to patch multiples, and odd row pitches (the byte-load path)."""
    lut = _im2col_domain(cuda)
    g = torch.Generator(device=cuda).manual_seed(B + H)
    img = torch.randint(0, 256, (B, H, W, 3), generator=g, device=cuda, dtype=torch.uint8)
    out = _im2col(img, P)
    Hp, Wp = H // P, W // P
    ch = torch.arange(3, device=cuda)
    step = 24
    for b0 in range(0, B, step):
        part = img[b0:b0 + step, :Hp * P, :Wp * P].long()
        nb = part.shape[0]
        want = lut[ch, part].view(nb, Hp, P, Wp, P, 3).permute(0, 1, 3, 5, 2, 4).reshape(nb * Hp * Wp, 3 * P * P)
        got = out[b0 * Hp * Wp:(b0 + nb) * Hp * Wp]
        assert torch.equal(got, want), f"images {b0}..{b0 + nb - 1}: {_diff(got != want)}"


def _ln_inputs(M, d, g, dev):
    """LayerNorm rows in repeating groups of 1024: N(0.5, 3^2) in [0, 256), a common offset of 1e3 in [256, 512) and
    of -2e3 in [512, 640), one outlier channel (x 50) per row in [640, 896), tiny rows (x 1e-3) in [896, 1024)."""
    x = torch.randn(M, d, generator=g, device=dev) * 3 + 0.5
    i = torch.arange(M, device=dev) % 1024
    up = ((i >= 256) & (i < 512)).nonzero()[:, 0]
    x[up] = 1e3 + torch.randn(up.numel(), d, generator=g, device=dev)
    down = ((i >= 512) & (i < 640)).nonzero()[:, 0]
    x[down] = -2e3 + torch.randn(down.numel(), d, generator=g, device=dev)
    r = ((i >= 640) & (i < 896)).nonzero()[:, 0]
    x[r, (r * 7) % d] *= 50.0                                    # one outlier channel per row
    x[i >= 896] *= 1e-3
    return x


def _ln_bound(x, gamma, beta, eps):
    """float64 LayerNorm y of fp32 rows x and the bound on |y_kernel - y| (see test_layernorm_float64_bound):
    (y, fp32 allowance pre, bound = pre + half an fp16 ulp)."""
    x64, g64, b64 = x.double(), gamma.double(), beta.double()
    mu = x64.mean(-1, keepdim=True)
    xc = x64 - mu
    sig = torch.sqrt((xc * xc).mean(-1, keepdim=True) + eps)
    y = xc / sig * g64 + b64
    pre = (g64.abs() * (16 * 2.0 ** -23 * xc.abs() + 16 * 2.0 ** -24 * x64.abs().mean(-1, keepdim=True)) / sig
           + 2.0 ** -23 * ((xc / sig * g64).abs() + b64.abs()))
    return y, pre, pre + 0.5 * _ulp16(y.abs() + pre)


@pytest.mark.parametrize("d", [384, 768])
def test_layernorm_float64_bound(cuda, d):
    """Bound per element: half an fp16 ulp of y, plus |gamma| / sigma times (16 2^-23 |x - mu| for the variance,
    rsqrt and products, and 16 2^-24 mean|x| for the fp32 mean), plus 2^-23 (|gamma xhat| + |beta|). Rows with a
    common offset of 1e3 or -2e3 break a one-pass variance E[x^2] - mu^2 by orders of magnitude more than this."""
    _l, lib = _lib()
    M = 1024
    g = torch.Generator(device=cuda).manual_seed(d)
    x = _ln_inputs(M, d, g, cuda)
    gamma = torch.randn(d, generator=g, device=cuda)
    beta = torch.randn(d, generator=g, device=cuda)
    eps = 1e-6
    buf = _out_buffer(M, d, torch.float16, cuda)
    _l.check(lib.dss_op_layernorm_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), buf.data_ptr(), M, d, eps,
                                      _l.stream_ptr()), "layernorm")
    torch.cuda.synchronize()
    _assert_guard(buf, M)
    y, pre, bound = _ln_bound(x, gamma, beta, eps)
    err = (buf[:M].double() - y).abs()
    ok = err <= bound
    # half an ulp is the rounding of a correct value: report the share of the fp32 allowance used beyond it
    print(f"layernorm d={d}: worst (err - 0.5 ulp16) / fp32 allowance {float(((err - (bound - pre)) / pre).max()):.3f}")
    assert ok.all(), f"layernorm beyond its rounding bound: {_diff(~ok)}"
