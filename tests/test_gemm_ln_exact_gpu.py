"""-m gpu: the LayerNorm-fused GEMM (csrc/gemm_ln.cu, dss_op_gemm_ln_f16) checked exactly.

Its A operand never leaves shared memory: three producer warps normalise the rows and write them by hand into the 128 B
swizzled panel, for row blocks paired across a 2-CTA cluster, and the panel is turned over once per unit. So it is
checked through the output:

  - Integer rows x = m + a s (s a balanced +-1 pattern, m a multiple of 2^-3, a a power of two) have exact fp32 row
    sums and normalise to +-1 within about 2^-15; with integer gamma and beta (|beta| != |gamma| unless gamma = 0, so
    that no element lands near 0, where fp16 would keep the noise) the A operand is exactly the integer gamma s + beta,
    the integer weights make every accumulator an integer below 2^24, and the output is compared bit for bit.
  - One-hot weights copy the panel to the output element by element: it must be bitwise the stand-alone LayerNorm
    kernel's output on the same x (the claim of gemm_ln.cu's header) and lie within that kernel's float64 bound.
  - On general data the fused kernel equals LayerNorm followed by the plain GEMM bit for bit.

Outputs are NaN-filled and followed by sentinel rows that must stay untouched."""
import pytest
import torch

from conftest import load_pkg
from test_vit_exact_gpu import GELU_ERR, _assert_guard, _diff, _ln_bound, _ln_inputs, _out_buffer, _ulp16

pytestmark = pytest.mark.gpu

K = 384
EPS = 1e-6
BENCH_ROWS = 264 * 901        # the benchmark's qkv / fc1 rows: 264 images of 901 tokens
ROWS = ["1", "127", "128", "129", "257", "sms128-1", "sms128+1", "bench"]
COLS = [128, 256, 384, 640, 1152, 1536]   # tile width 128 (1, 2, 5 n-tiles) and 192 (2, 6, 8 n-tiles)


def _lib():
    _l = load_pkg("_lib")
    return _l, _l.load()


def _rows(name, dev):
    """M = 257: the last unit's second (rank-1) row block lies wholly past M. SMs x 128 rows give every cluster exactly
    one unit (of two row blocks); one row more gives one cluster a second unit."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    return {"sms128-1": sms * 128 - 1, "sms128+1": sms * 128 + 1, "bench": BENCH_ROWS}.get(name) or int(name)


def _gemm_ln(x, gamma, beta, Wt, bias, gelu):
    _l, lib = _lib()
    M, N = x.shape[0], Wt.shape[0]
    buf = _out_buffer(M, N, torch.float16, x.device)
    _l.check(lib.dss_op_gemm_ln_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), Wt.data_ptr(), bias.data_ptr(),
                                    buf.data_ptr(), M, N, K, EPS, int(gelu), _l.stream_ptr()), "gemm_ln")
    torch.cuda.synchronize()
    _assert_guard(buf, M)
    return buf[:M]


def _layernorm(x, gamma, beta):
    _l, lib = _lib()
    M = x.shape[0]
    buf = _out_buffer(M, K, torch.float16, x.device)
    _l.check(lib.dss_op_layernorm_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), buf.data_ptr(), M, K, EPS,
                                      _l.stream_ptr()), "layernorm")
    torch.cuda.synchronize()
    _assert_guard(buf, M)
    return buf[:M]


def _chunks(M, N):
    step = max(128, (1 << 24) // N)
    return [(r0, min(M, r0 + step)) for r0 in range(0, M, step)]


# ---------------------------------------------------------------------------------------------------------------
# bit for bit on integer rows

def _integer_operands(M, N, gelu, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    s = torch.where(torch.rand(M, K, generator=g, device=dev).argsort(1) < K // 2, 1.0, -1.0)   # 192 of each sign
    m = torch.randint(-512, 513, (M, 1), generator=g, device=dev).float() * 2.0 ** -3
    a = torch.exp2(torch.randint(-2, 4, (M, 1), generator=g, device=dev).float())
    x = (m + a * s).contiguous()
    gamma = torch.randint(-4, 5, (K,), generator=g, device=dev).float()
    beta = torch.randint(-8, 9, (K,), generator=g, device=dev).float()
    beta[(gamma != 0) & (beta.abs() == gamma.abs())] += 1.0     # no A element of 0 from gamma s + beta
    Wt = torch.randint(-8, 9, (N, K), generator=g, device=dev).float()
    if gelu:   # accumulators: multiples of 2^-6 that densely cover [-10, 10]
        Wt = Wt * 2.0 ** -6
        bias = torch.randint(-128, 129, (N,), generator=g, device=dev).float() * 2.0 ** -6
    else:      # integers up to 384 * 12 * 8: above 2048 fp16 rounds them to even
        bias = torch.randint(-8, 9, (N,), generator=g, device=dev).float()
    A = gamma[None, :] * s + beta[None, :]                       # what the panel must hold, exactly
    return x, gamma, beta, Wt.half(), bias, A


@pytest.mark.parametrize("gelu", [0, 1])
@pytest.mark.parametrize("N", COLS)
@pytest.mark.parametrize("rows", ROWS)
def test_integer_rows_bit_for_bit(cuda, rows, N, gelu):
    M = _rows(rows, cuda)
    x, gamma, beta, Wt, bias, A = _integer_operands(M, N, gelu, seed=M * 7 + N + gelu, dev=cuda)
    out = _gemm_ln(x, gamma, beta, Wt, bias, gelu)
    Wt64, b64 = Wt.double().T.contiguous(), bias.double()
    worst_gelu = 0.0
    for r0, r1 in _chunks(M, N):
        ref = torch.addmm(b64, A[r0:r1].double(), Wt64)           # exact: multiples of 2^-6 far below 2^53
        got = out[r0:r1]
        if gelu:
            gl = ref * 0.5 * (1.0 + torch.erf(ref * (0.5 ** 0.5)))
            g64 = got.double()
            err = (g64 - gl).abs()
            bound = 0.5 * _ulp16(torch.maximum(gl.abs(), g64.abs())) + GELU_ERR
            bad = ~(err <= bound)
            assert not bad.any(), f"M={M} N={N} GELU beyond 0.5 ulp16 + {GELU_ERR}: {_diff(bad, r0)}"
            worst_gelu = max(worst_gelu, float(((err - (bound - GELU_ERR)) / GELU_ERR).max()))
        else:
            want = ref.half()                                      # an integer below 2^24: one rounding to fp16
            if not torch.equal(got, want):
                bad = got != want
                raise AssertionError(f"M={M} N={N}: {_diff(bad, r0)}; got {got[bad][:4].tolist()} "
                                     f"want {want[bad][:4].tolist()}")
    if gelu:
        print(f"gemm_ln gelu M={M} N={N}: worst (err - 0.5 ulp16) / {GELU_ERR} = {worst_gelu:.3f}")


# ---------------------------------------------------------------------------------------------------------------
# the A panel itself, through one-hot weights

@pytest.mark.parametrize("N", [384, 640])
@pytest.mark.parametrize("rows", ["129", "257", "sms128+1", "bench"])
def test_panel_is_the_layernorm_kernel_output(cuda, rows, N):
    """Wt[n] = e_pi(n) (pi: random permutations of the 384 columns, concatenated), zero bias, no GELU: out[r, n] =
    A[r, pi(n)] exactly. The panel must be bitwise dss_op_layernorm_f16 on the same x, and within its float64 bound.
    x: offsets of 1e3 and -2e3, an outlier channel, tiny rows (test_layernorm_float64_bound's rows)."""
    M = _rows(rows, cuda)
    g = torch.Generator(device=cuda).manual_seed(M + N)
    x = _ln_inputs(M, K, g, cuda)
    gamma = torch.randn(K, generator=g, device=cuda)
    beta = torch.randn(K, generator=g, device=cuda)
    perm = torch.cat([torch.randperm(K, generator=g, device=cuda) for _ in range((N + K - 1) // K)])[:N]
    Wt = torch.zeros(N, K, device=cuda, dtype=torch.float16)
    Wt[torch.arange(N, device=cuda), perm] = 1.0
    bias = torch.zeros(N, device=cuda)
    out = _gemm_ln(x, gamma, beta, Wt, bias, 0)
    first = torch.empty(K, dtype=torch.long, device=cuda)
    first[perm[:K]] = torch.arange(K, device=cuda)              # the output column n < K that holds panel column c
    panel = out[:, first]
    assert torch.equal(out, panel[:, perm]), "one-hot columns copying the same panel column differ"
    ln = _layernorm(x, gamma, beta)
    if not torch.equal(panel, ln):
        bad = panel != ln
        ulps = ((panel.double() - ln.double()).abs() / _ulp16(torch.maximum(panel.double().abs(), ln.double().abs())))
        raise AssertionError(f"M={M} N={N}: the fused panel is not the LayerNorm kernel's output: {_diff(bad)}, "
                             f"up to {float(ulps.max()):.1f} fp16 ulp")
    worst = 0.0
    for r0, r1 in _chunks(M, K):
        y, pre, bound = _ln_bound(x[r0:r1], gamma, beta, EPS)
        err = (panel[r0:r1].double() - y).abs()
        ok = err <= bound
        assert ok.all(), f"M={M}: panel beyond the LayerNorm float64 bound: {_diff(~ok, r0)}"
        worst = max(worst, float(((err - (bound - pre)) / pre).max()))
    print(f"gemm_ln panel M={M} N={N}: bitwise the LayerNorm kernel; worst (err - 0.5 ulp16) / fp32 allowance "
          f"{worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------
# fused against the two-kernel path on general data

@pytest.mark.parametrize("gelu", [0, 1])
@pytest.mark.parametrize("N", [384, 1152, 1536])
@pytest.mark.parametrize("rows", ["129", "sms128+1", "bench"])
def test_fused_matches_layernorm_then_gemm(cuda, rows, N, gelu):
    """Same A operand, same K order of the wgmma steps, same epilogue: the same bits as the two-kernel path."""
    _l, lib = _lib()
    M = _rows(rows, cuda)
    g = torch.Generator(device=cuda).manual_seed(3 * M + N + gelu)
    x = _ln_inputs(M, K, g, cuda)
    gamma = torch.randn(K, generator=g, device=cuda) * 0.5 + 1.0
    beta = torch.randn(K, generator=g, device=cuda) * 0.2
    Wt = (torch.randn(N, K, generator=g, device=cuda) * 0.05).half()
    bias = torch.randn(N, generator=g, device=cuda) * 0.1
    fused = _gemm_ln(x, gamma, beta, Wt, bias, gelu)
    y = _layernorm(x, gamma, beta)
    two = _out_buffer(M, N, torch.float16, cuda)
    _l.check(lib.dss_op_gemm_f16(y.data_ptr(), Wt.data_ptr(), bias.data_ptr(), two.data_ptr(), M, N, K,
                                 _l.EPI_BIAS_GELU_F16 if gelu else _l.EPI_BIAS_F16, None, 0, 0, _l.stream_ptr()), "gemm")
    torch.cuda.synchronize()
    _assert_guard(two, M)
    two = two[:M]
    assert torch.isfinite(fused).all()
    worst, ndiff = 0.0, 0
    for r0, r1 in _chunks(M, N):
        a, b = fused[r0:r1].double(), two[r0:r1].double()
        d = (a - b).abs() / _ulp16(torch.maximum(a.abs(), b.abs()))
        worst = max(worst, float(d.max()))
        ndiff += int((fused[r0:r1] != two[r0:r1]).sum())
    print(f"gemm_ln vs layernorm + gemm M={M} N={N} gelu={gelu}: {ndiff} of {M * N} outputs differ, "
          f"largest difference {worst:.1f} fp16 ulp")
    assert ndiff == 0, f"M={M} N={N} gelu={gelu}: {ndiff} outputs differ, by up to {worst:.1f} fp16 ulp"
