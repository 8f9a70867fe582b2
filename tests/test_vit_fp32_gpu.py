"""-m gpu: the fp32-precision ViT (DinoViT(..., precision="fp32"), split-fp16 operands) against float64.

Every tensor-core operand is split as x = hi + lo into hi, hi/64 and 64 lo (fp16); one fp16 product over the three groups
is hi hi' + hi lo' + lo hi'. Bound of one such GEMM against float64 (DESIGN.md section 3), per output element:
    |c - c64| <= (3 * 2^-22 + 2^-23 * (K' / 16 + 2)) * sum_k |a_k| |b_k|      (K' = 3 K)
the first term the split (dropped lo lo', rounding of 64 lo), the second the fp32 accumulation of the K' / 16 wgmma
k-steps. A plain fp16 product misses it by about 2^-11 and fails it (checked below, so the bound discriminates)."""
import numpy as np
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

EPS_SPLIT = 3 * 2.0 ** -22


def _gemm_bound(K):
    return EPS_SPLIT + 2.0 ** -23 * (3 * K / 16 + 2)


def _lib():
    return load_pkg("_lib")


def _split(x, order):
    L = _lib()
    rows, cols = x.shape
    out = torch.empty(rows, 3 * cols, dtype=torch.float16, device=x.device)
    L.check(L.load().dss_op_split_f16(x.data_ptr(), out.data_ptr(), rows, cols, order, L.stream_ptr()), "split")
    return out


def _gemm(A16, W16, bias, out, M, N, K, epi, aux=None, rin=0, rout=0):
    L = _lib()
    L.check(L.load().dss_op_gemm_f16(A16.data_ptr(), W16.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K, epi,
                                     L.ptr(aux), rin, rout, L.stream_ptr()), "gemm")
    torch.cuda.synchronize()
    return out


def _operands(M, N, K, seed, dev):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    A[:, :4] *= 50.0                                     # outlier channels, as the fp16 path's overflow tests use
    W = torch.randn(N, K, generator=g) * 0.02
    W[:, -8:] = torch.linspace(1e-4, 1e-3, 8)            # small weights: the hi/64 and 64 lo subnormal floor
    bias = torch.randn(N, generator=g) * 0.1
    return A.to(dev), W.to(dev), bias.to(dev)


@pytest.mark.parametrize("K", [384, 768, 1536, 3072, 3 * 16 * 16, 3 * 8 * 8])
@pytest.mark.parametrize("epi", ["BIAS_F32", "BIAS_RESID_F32", "PATCH_F32", "DROPCLS_F32"])
def test_split_gemm_against_float64(cuda, K, epi):
    L = _lib()
    M, N = 394, 384
    A, W, bias = _operands(M, N, K, 7 + K, cuda)
    A64, W64 = A.double(), W.double()
    acc64 = A64 @ W64.T + bias.double()
    mag = A64.abs() @ W64.abs().T + bias.double().abs()
    As, Ws = _split(A, 0), _split(W, 1)
    if epi in ("BIAS_F32", "BIAS_RESID_F32"):
        code = L.EPI_BIAS_F32 if epi == "BIAS_F32" else L.EPI_BIAS_RESID_F32
        resid = torch.randn(M, N, device=cuda) if epi == "BIAS_RESID_F32" else torch.zeros(M, N, device=cuda)
        out = _gemm(As, Ws, bias, resid.clone(), M, N, 3 * K, code)
        want, mag = acc64 + resid.double(), mag + resid.double().abs()
        got = out.double()
    elif epi == "PATCH_F32":
        Np = 197 - 1
        T = Np + 1
        B = -(-M // Np)
        Ap = torch.cat([A, A[: B * Np - M]]) if B * Np > M else A
        Mp = B * Np
        aux = torch.randn(T, N, device=cuda)
        out = _gemm(_split(Ap, 0), Ws, bias, torch.zeros(B * T, N, device=cuda), Mp, N, 3 * K, L.EPI_PATCH_F32, aux, Np, T)
        acc64 = Ap.double() @ W64.T + bias.double()
        mag = Ap.double().abs() @ W64.abs().T + bias.double().abs()
        idx = torch.arange(Mp, device=cuda)
        rows = (idx // Np) * T + idx % Np + 1
        got = out.double()[rows]
        want = acc64 + aux.double()[idx % Np + 1]
        mag = mag + aux.double().abs()[idx % Np + 1]
    else:
        T = 197
        B = M // T
        Md = B * T
        out = _gemm(As[:Md].contiguous(), Ws, bias, torch.zeros(B * (T - 1), N, device=cuda), Md, N, 3 * K,
                    L.EPI_DROPCLS_F32, None, T, T - 1)
        idx = torch.arange(Md, device=cuda)
        keep = idx % T != 0
        rows = (idx // T) * (T - 1) + idx % T - 1
        got, want, mag = out.double()[rows[keep]], acc64[:Md][keep], mag[:Md][keep]
    ratio = ((got - want).abs() / (_gemm_bound(K) * mag)).max().item()
    print(f"split GEMM K={K} {epi}: max |err| / bound = {ratio:.3f}")
    assert torch.isfinite(got).all()
    assert ratio <= 1.0, ratio


def test_split_gemm_bound_rejects_plain_fp16(cuda):
    """The bound is tight enough to tell a split product from an fp16 one (and from weights packed in A order)."""
    L = _lib()
    M, N, K = 256, 384, 768
    A, W, bias = _operands(M, N, K, 3, cuda)
    mag = A.double().abs() @ W.double().abs().T + bias.double().abs()
    want = A.double() @ W.double().T + bias.double()
    plain = _gemm(A.half(), W.half(), bias, torch.zeros(M, N, device=cuda), M, N, K, L.EPI_BIAS_F32)
    a_order = _gemm(_split(A, 0), _split(W, 0), bias, torch.zeros(M, N, device=cuda), M, N, 3 * K, L.EPI_BIAS_F32)
    for name, got in (("fp16", plain), ("weights in A order", a_order)):
        ratio = ((got.double() - want).abs() / (_gemm_bound(K) * mag)).max().item()
        print(f"{name}: max |err| / bound = {ratio:.1f}")
        assert ratio > 2.0, (name, ratio)


def _groups(y, n):
    """split output [rows, 3n] -> (hi, hi/64, 64 lo) as float64"""
    y = y.double()
    return y[:, :n], y[:, n:2 * n], y[:, 2 * n:]


def _check_groups(y, v32, n):
    """hi = fp16(v), the second group = fp16(hi / 64) exactly; hi + (64 lo) / 64 is v to the 2^-22 of the rounded
    64 lo (plus the fp16 subnormal floor 2^-25 / 64)."""
    hi, his, los = _groups(y, n)
    assert torch.equal(hi, v32.half().double())
    assert torch.equal(his, (hi / 64).half().double())
    err = (hi + los / 64 - v32.double()).abs()
    assert (err <= 2.0 ** -22 * v32.double().abs() + 2.0 ** -31).all(), err.max().item()


@pytest.mark.parametrize("d", [384, 768])
def test_layernorm_split(cuda, d):
    L = _lib()
    M = 333
    g = torch.Generator(device="cpu").manual_seed(d)
    x = (torch.randn(M, d, generator=g) * 3 + 1).to(cuda)
    x[:, 5] *= 50.0
    gamma = (1 + 0.1 * torch.randn(d, generator=g)).to(cuda)
    beta = (0.1 * torch.randn(d, generator=g)).to(cuda)
    y = torch.empty(M, 3 * d, dtype=torch.float16, device=cuda)
    L.check(L.load().dss_op_layernorm_split_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), M, d,
                                                1e-6, L.stream_ptr()))
    # the split value's hi is the fp16 path's output: same statistics, same rounding
    y16 = torch.empty(M, d, dtype=torch.float16, device=cuda)
    L.check(L.load().dss_op_layernorm_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y16.data_ptr(), M, d, 1e-6,
                                          L.stream_ptr()))
    torch.cuda.synchronize()
    hi, his, los = _groups(y, d)
    assert torch.equal(hi, y16.double())
    assert torch.equal(his, (hi / 64).half().double())
    v = hi + los / 64
    ln64 = torch.nn.functional.layer_norm(x.double(), (d,), gamma.double(), beta.double(), 1e-6)
    err = (v - ln64).abs().max().item()
    print(f"layernorm split d={d}: max |err| vs float64 {err:.2e}")
    assert err <= 2e-6 * (ln64.abs().max().item() + 1)


def test_gelu_split(cuda):
    L = _lib()
    M, n = 257, 1536
    h = (torch.randn(M, n, generator=torch.Generator().manual_seed(1)) * 3).to(cuda)
    y = torch.empty(M, 3 * n, dtype=torch.float16, device=cuda)
    L.check(L.load().dss_op_gelu_split_f16(h.data_ptr(), y.data_ptr(), M, n, L.stream_ptr()))
    torch.cuda.synchronize()
    hi, his, los = _groups(y, n)
    assert torch.equal(his, (hi / 64).half().double())
    g64 = torch.nn.functional.gelu(h.double())
    err = (hi + los / 64 - g64).abs()
    # erff and the fp32 products: a few ulp of gelu, plus 1 + erf cancelling for negative x (~1e-7 |x|)
    tol = 1e-6 * g64.abs() + 2e-7 * h.double().abs() + 2.0 ** -31
    print(f"gelu split: max |err| / tol = {(err / tol).max().item():.3f}")
    assert (err <= tol).all()


@pytest.mark.parametrize("H,W,pad", [(224, 224, 0), (100, 132, 0), (100, 132, 1), (37, 50, 1)])
@pytest.mark.parametrize("P", [16, 8])
def test_im2col_split(cuda, H, W, pad, P):
    from oracle import dino_vit
    L = _lib()
    synth = load_pkg("synth")
    B = 2
    imgs = synth.blobs_batch(B, H, W, 5).to(cuda)
    Hp, Wp = (-(-H // P), -(-W // P)) if pad else (H // P, W // P)
    Kp = 3 * P * P
    out = torch.empty(B * Hp * Wp, 3 * Kp, dtype=torch.float16, device=cuda)
    L.check(L.load().dss_op_im2col_split_f16(imgs.data_ptr(), out.data_ptr(), B, H, W, P, pad, L.stream_ptr()))
    torch.cuda.synchronize()
    v = []
    for b in range(B):
        x = dino_vit.preprocess_u8(imgs[b].cpu(), P) if not pad else None
        if pad:
            t = imgs[b].cpu().permute(2, 0, 1).float() / 255.0
            mean = torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)
            std = torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)
            t = (t - mean) / std
            x = torch.zeros(1, 3, Hp * P, Wp * P)
            x[0, :, :H, :W] = t
        v.append(x[0].unfold(1, P, P).unfold(2, P, P).permute(1, 2, 0, 3, 4).reshape(Hp * Wp, Kp))
    _check_groups(out, torch.cat(v).to(cuda), Kp)


def _attention_split(qkv, B, T, heads):
    L = _lib()
    d = 64 * heads
    scratch = torch.empty(B * T, 9 * d, dtype=torch.float16, device=qkv.device)
    out = torch.empty(B * T, 3 * d, dtype=torch.float16, device=qkv.device)
    L.check(L.load().dss_op_attention_split_f16(qkv.data_ptr(), scratch.data_ptr(), out.data_ptr(), B, T, heads,
                                                L.stream_ptr()), "attention_split")
    torch.cuda.synchronize()
    hi, _, los = _groups(out, d)
    return (hi + los / 64).view(B, T, d)


def _attention_check(qkv, o, B, T, heads):
    """per element: |o - o64| <= (2^-18 a + 2^-20) (P |V|) + 2^-22 |o|, a = max_j sum |q||k| / 8 of the row (the
    split score error and its fp32 accumulation), P |V| the softmax-weighted magnitude of the values"""
    d = 64 * heads
    x = qkv.view(B, T, 3, heads, 64).double()
    worst = 0.0
    for b in range(B):
        for h in range(heads):
            q, k, v = x[b, :, 0, h], x[b, :, 1, h], x[b, :, 2, h]
            p = torch.softmax(q @ k.T / 8, dim=-1)
            o64 = p @ v
            a = ((q.abs() @ k.abs().T) / 8).max(dim=-1, keepdim=True).values
            tol = (2.0 ** -18 * a + 2.0 ** -20) * (p @ v.abs()) + 2.0 ** -22 * o64.abs()
            got = o[b, :, h * 64:(h + 1) * 64]
            worst = max(worst, ((got - o64).abs() / tol).max().item())
    return worst


@pytest.mark.parametrize("T,heads", [(197, 6), (901, 6), (3601, 12), (6401, 12), (528, 6), (713, 12), (962, 6)])
def test_attention_split_against_float64(cuda, T, heads):
    B = 2 if T < 3000 else 1
    d = 64 * heads
    g = torch.Generator().manual_seed(T + heads)
    qkv = (torch.randn(B * T, 3 * d, generator=g) * 1.5).to(cuda)
    o = _attention_split(qkv, B, T, heads)
    assert torch.isfinite(o).all()
    worst = _attention_check(qkv, o, B, T, heads)
    print(f"split attention T={T} heads={heads}: max |err| / bound = {worst:.3f}")
    assert worst <= 1.0


def test_attention_split_dominating_and_equal_scores(cuda):
    B, T, heads = 2, 197, 6
    d = 64 * heads
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B * T, 3 * d, generator=g)
    qkv[:T, :64] = 0.0                                   # image 0, head 0: every score equal (uniform attention)
    qkv[T:, :64] = 2.0                                   # image 1, head 0: key 5 dominates every query
    qkv[T + 5, d:d + 64] = 8.0
    qkv = qkv.to(cuda)
    o = _attention_split(qkv, B, T, heads)
    worst = _attention_check(qkv, o, B, T, heads)
    print(f"dominating / equal scores: max |err| / bound = {worst:.3f}")
    assert worst <= 1.0


def test_attention_split_batch_equals_solo(cuda):
    B, T, heads = 3, 901, 6
    qkv = torch.randn(B * T, 3 * 64 * heads, generator=torch.Generator().manual_seed(4)).to(cuda)
    o = _attention_split(qkv, B, T, heads)
    for b in range(B):
        solo = _attention_split(qkv[b * T:(b + 1) * T].contiguous(), 1, T, heads)
        assert torch.equal(o[b], solo[0]), b


# ---- the whole ViT
# The fp32-mode K features may be at most this many times further from float64 than the fp32 oracle's. Measured on an
# H100 80GB HBM3 (700 W): 5.1-5.3 for ViT-S/16 (T = 197 ... 901), 12.9 for ViT-B/8 at 480^2 (T = 3601) and 18.4 at 640^2
# (T = 6401): the wgmma accumulation rounds once per 16-key step of P V and per 16 channels of each GEMM, where the
# oracle's fp32 products accumulate in longer FMA chains. Bounds: 1.5x the measured ratio.
FEATURE_FACTOR = {"dino_vits16": 8.0, "dino_vitb8": 28.0}


@pytest.fixture(scope="module")
def vits16(cuda):
    from oracle import dino_vit
    vit = load_pkg("vit")
    ref = dino_vit.build("dino_vits16", seed=0)
    sd = ref.state_dict()
    return ref.to(cuda).eval(), vit.DinoViT("dino_vits16", sd, device=cuda, precision="fp32"), sd


def _feature_errors(ref, mine, imgs, P, cuda):
    from oracle import dino_vit
    import copy
    ref64 = copy.deepcopy(ref).double()
    x = torch.cat([dino_vit.preprocess_u8(im, P) for im in imgs]).to(cuda)
    k64 = ref64.forward_k(x.double())
    k32 = ref.forward_k(x)
    k = mine.forward_k(imgs.to(cuda))
    torch.cuda.synchronize()
    rel = lambda a: ((a.double() - k64).norm() / k64.norm()).item()   # noqa: E731
    return rel(k), rel(k32)


@pytest.mark.parametrize("H,W,B", [(224, 224, 2), (480, 480, 2), (375, 500, 2)])
def test_features_vits16(cuda, vits16, H, W, B):
    ref, mine, _ = vits16
    synth = load_pkg("synth")
    e_split, e_ref = _feature_errors(ref, mine, synth.blobs_batch(B, H, W, 21), 16, cuda)
    print(f"ViT-S/16 {H}x{W}: fp32-mode rel-L2 vs float64 {e_split:.3e}, fp32 oracle {e_ref:.3e}, "
          f"ratio {e_split / e_ref:.2f}")
    assert e_split <= FEATURE_FACTOR["dino_vits16"] * e_ref


@pytest.mark.parametrize("H,W", [(480, 480), (640, 640)])
def test_features_vitb8(cuda, H, W):
    from oracle import dino_vit
    vit = load_pkg("vit")
    synth = load_pkg("synth")
    ref = dino_vit.build("dino_vitb8", seed=0)
    mine = vit.DinoViT("dino_vitb8", ref.state_dict(), device=cuda, precision="fp32")
    e_split, e_ref = _feature_errors(ref.to(cuda).eval(), mine, synth.blobs_batch(1, H, W, 31), 8, cuda)
    print(f"ViT-B/8 {H}x{W}: fp32-mode rel-L2 vs float64 {e_split:.3e}, fp32 oracle {e_ref:.3e}, "
          f"ratio {e_split / e_ref:.2f}")
    assert e_split <= FEATURE_FACTOR["dino_vitb8"] * e_ref


def _evec_err(v, vo):
    """worst sign-aligned rel-L2 over eigenvectors 1..4 (vector 0 is the constant one)"""
    v, vo = np.asarray(v, np.float64), np.asarray(vo, np.float64)
    return max(np.linalg.norm(v[k] - (np.sign(np.dot(v[k], vo[k])) or 1.0) * vo[k]) / np.linalg.norm(vo[k])
               for k in range(1, 5))


def test_end_to_end_eigenvectors(cuda, vits16):
    """16 blobs images at 480^2, K = 5: images -> fp32-mode features -> the library's eigensolver, against the
    reference route (fp32 oracle ViT + scipy eigensolver). An image over 1e-4 is attributed as bench.py does: both
    routes against a float64 eigensolve of the float64 oracle's features; it passes only if the reference route is the
    one further off. The fp16 mode's figure is printed beside it."""
    import copy
    from oracle import dino_vit, eigs_ref
    pipeline = load_pkg("pipeline")
    vit = load_pkg("vit")
    synth = load_pkg("synth")
    ref, mine, sd = vits16
    imgs = synth.blobs_batch(16, 480, 480, seed0=100)
    mine16 = vit.DinoViT("dino_vits16", sd, device=cuda)
    ref64 = copy.deepcopy(ref).double()
    x = [dino_vit.preprocess_u8(imgs[b], 16).to(cuda) for b in range(16)]
    vec_ref = [eigs_ref.extract_eig(ref.forward_k(x[b])[0].cpu(), 5, rng_seed=0)[1].numpy() for b in range(16)]
    for name, model in (("fp32", mine), ("fp16", mine16)):
        pipe = pipeline.SpectralPipeline("dino_vits16", K=5, device=cuda, model=model, vit_batch=8)
        _, evecs, info = pipe.run_host(imgs.pin_memory())
        errs = [_evec_err(evecs[b].numpy(), vec_ref[b]) for b in range(16)]
        assert all(int(info[b, 1]) == 1 for b in range(16))
        print(f"{name} mode: sign-aligned eigenvector rel-L2 vs the reference route, worst {max(errs):.2e}, "
              f"median {float(np.median(errs)):.2e}")
        if name == "fp16":
            continue
        for b in (b for b in range(16) if errs[b] > 1e-4):
            vec64 = eigs_ref.eigh_f64(ref64.forward_k(x[b].double())[0].cpu(), 6)[1][:5]
            ours, theirs = _evec_err(evecs[b].numpy(), vec64), _evec_err(vec_ref[b], vec64)
            print(f"image {b}: {errs[b]:.2e} over 1e-4; vs float64: ours {ours:.2e}, reference route {theirs:.2e}")
            assert theirs > ours, (b, ours, theirs)


def test_forward_last_and_cls_attention(cuda, vits16):
    """Localization outputs in fp32 mode: the k third equals forward_k's bits (crop), q / v and the CLS attention row
    against the float64 oracle's last block."""
    import copy
    from oracle import dino_vit
    ref, mine, _ = vits16
    synth = load_pkg("synth")
    imgs = synth.blobs_batch(2, 224, 224, 3).to(cuda)
    f, _ = mine.forward_last(imgs, which="k", pad=False)
    assert torch.equal(f, mine.forward_k(imgs))
    ref64 = copy.deepcopy(ref).double()
    x = torch.cat([dino_vit.preprocess_u8(im.cpu(), 16) for im in imgs]).to(cuda).double()
    tok = ref64.forward_tokens(x, 11)
    blk = ref64.blocks[11]
    qkv = blk.attn.qkv(blk.norm1(tok))
    d, heads = 384, 6
    for w, which in enumerate("qkv"):
        got, att = mine.forward_last(imgs, which=which, pad=False, cls_attn=True)
        want = qkv[:, 1:, w * d:(w + 1) * d]
        rel = ((got.double() - want).norm() / want.norm()).item()
        print(f"forward_last {which}: rel-L2 vs float64 {rel:.2e}")
        assert rel <= 1e-5
    q = qkv[:, 0, :d].view(2, heads, 64)
    k = qkv[:, :, d:2 * d].view(2, -1, heads, 64)
    a64 = torch.softmax(torch.einsum("bhc,bthc->bht", q, k) / 8, dim=-1)[:, :, 1:]
    err = (att.double() - a64).abs().max().item()
    print(f"CLS attention: max |err| vs float64 {err:.2e}")
    assert err <= 1e-6


def _oracle_last(ref, imgs, cuda):
    """fp32 oracle: last block's qkv [B, T, 3d] and CLS attention [B, heads, N]"""
    from oracle import dino_vit
    x = torch.cat([dino_vit.preprocess_u8(im.cpu(), 16) for im in imgs]).to(cuda)
    tok = ref.forward_tokens(x, 11)
    blk = ref.blocks[11]
    qkv = blk.attn.qkv(blk.norm1(tok))
    B, d, heads = imgs.shape[0], 384, 6
    q = qkv[:, 0, :d].reshape(B, heads, 64)
    k = qkv[:, :, d:2 * d].reshape(B, -1, heads, 64)
    return qkv, torch.softmax(torch.einsum("bhc,bthc->bht", q, k) / 8, dim=-1)[:, :, 1:].contiguous()


def test_localization_boxes_match_fp32_oracle(cuda, vits16):
    """LOST (k features) and DINO-seg (CLS attention) boxes of fp32 mode equal those of the fp32 oracle's outputs."""
    ref, mine, _ = vits16
    loc = load_pkg("localize")
    synth = load_pkg("synth")
    imgs = synth.blobs_batch(4, 224, 224, 40).to(cuda)
    f, att = mine.forward_last(imgs, which="k", pad=True, cls_attn=True)
    qkv, att_ref = _oracle_last(ref, imgs, cuda)
    k_ref = qkv[:, 1:, 384:768].contiguous()
    got, want = loc.lost_boxes(f, (14, 14), (224, 224), 16), loc.lost_boxes(k_ref, (14, 14), (224, 224), 16)
    print("LOST boxes", got[0].tolist(), want[0].tolist())
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    got, want = loc.dinoseg_boxes(att, (14, 14), 16), loc.dinoseg_boxes(att_ref, (14, 14), 16)
    print("DINO-seg boxes", got[0].tolist(), want[0].tolist())
    assert np.array_equal(got[0], want[0])


# ---- interface
def test_default_equals_explicit_fp16(cuda, vits16):
    vit = load_pkg("vit")
    synth = load_pkg("synth")
    _, _, sd = vits16
    imgs = synth.blobs_batch(2, 224, 224, 9).to(cuda)
    a = vit.DinoViT("dino_vits16", sd, device=cuda).forward_k(imgs)
    b = vit.DinoViT("dino_vits16", sd, device=cuda, precision="fp16").forward_k(imgs)
    assert torch.equal(a, b)


def test_set_precision_after_load_refused(cuda, vits16):
    L = _lib()
    _, mine, _ = vits16
    rc = L.load().dss_vit_set_precision(mine._h, 0)
    assert rc == -1 and b"before dss_vit_load_weights" in L.load().dss_last_error()


def test_workspace_one_byte_short_refused(cuda, vits16):
    L = _lib()
    _, mine, _ = vits16
    lib = L.load()
    B, H, W = 1, 224, 224
    need = int(lib.dss_vit_workspace_bytes(mine._h, B, H, W))
    vit16 = load_pkg("vit").DinoViT("dino_vits16", vits16[2], device=cuda)
    assert need > int(lib.dss_vit_workspace_bytes(vit16._h, B, H, W))   # the split buffers are larger
    imgs = load_pkg("synth").blobs_batch(B, H, W, 0).to(cuda)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    out = torch.empty(B, 196, 384, device=cuda)
    rc = lib.dss_vit_forward_k(mine._h, imgs.data_ptr(), B, H, W, -1, out.data_ptr(), ws.data_ptr(), need - 1,
                               L.stream_ptr())
    assert rc == -3
    rc = lib.dss_vit_forward_k(mine._h, imgs.data_ptr(), B, H, W, -1, out.data_ptr(), ws.data_ptr(), need,
                               L.stream_ptr())
    assert rc == 0


def _write_dataset(tmp_path, n, H, W):
    from PIL import Image
    synth = load_pkg("synth")
    root = tmp_path / "images"
    root.mkdir()
    names = []
    for i in range(n):
        name = f"img_{i:03d}.png"
        Image.fromarray(synth.blobs_image(H, W, 70 + i).numpy()).save(root / name)
        names.append(name)
    (tmp_path / "list.txt").write_text("\n".join(names) + "\n")
    return root, tmp_path / "list.txt", names


def test_extract_commands_fp32(cuda, tmp_path, vits16):
    ex = load_pkg("extract")
    utils = load_pkg("extract_utils")
    vit = load_pkg("vit")
    root, lst, names = _write_dataset(tmp_path, 3, 112, 144)
    model = vit.DinoViT("dino_vits16", vit.random_state_dict("dino_vits16", 0), device=cuda, precision="fp32")
    ex.extract_features(str(lst), str(root), "dino_vits16", 2, str(tmp_path / "f"), seed=0, precision="fp32")
    ex.extract_all(str(lst), str(root), "dino_vits16", str(tmp_path / "fa"), str(tmp_path / "e"), K=4, batch_size=2,
                   seed=0, precision="fp32")
    for i, n in enumerate(names):
        img = torch.from_numpy(utils.read_image_rgb(root / n)).unsqueeze(0).to(cuda)
        k = model.forward_k(img).cpu()
        for fdir in ("f", "fa"):
            dct = torch.load(tmp_path / fdir / (n[:-4] + ".pth"), map_location="cpu")
            assert dct["k"].shape == (1, 7 * 9, 384) and dct["k"].dtype == torch.float32
            assert torch.equal(dct["k"], k), (fdir, n)
