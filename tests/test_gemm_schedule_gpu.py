"""-m gpu: the ping-pong GEMM schedule against the cooperative one, bit for bit (dss_debug_gemm_schedule).

Both schedules sum the same K slabs of every output element in the same order, so on the same seeded non-integer fp16
operands all four TMA-store epilogues must give identical bits. Cases: the benchmark's four ViT GEMMs at its 264-image
batch; M = 128 (the odd CTA's tile wholly out of bounds) and 129; an odd number of work items on every CTA pair; fewer
work items than CTA pairs; K = 8, 72, 384, 1536 (one zero-filled slab, a partial slab, the ring depth exceeded);
partial last n-tiles. Outputs are NaN-filled with guard sentinel rows after them: an element neither schedule writes
stays NaN and fails the comparison, and the guard rows must stay untouched."""
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

GUARD = 128
SENT = {torch.float32: -7777.25, torch.float16: -777.5}
EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RESID_F32, EPI_BIAS_F32 = range(4)
EPI_NAME = {EPI_BIAS_F16: "f16", EPI_BIAS_GELU_F16: "gelu", EPI_BIAS_RESID_F32: "resid", EPI_BIAS_F32: "f32"}
BENCH_M = 264 * 901


def _run(dev, epi, M, N, K, seed):
    _l = load_pkg("_lib")
    lib = _l.load()
    g = torch.Generator(device=dev).manual_seed(seed)
    A = torch.randn(M, K, generator=g, device=dev).half()
    Wt = (torch.randn(N, K, generator=g, device=dev) * K ** -0.5).half()
    bias = torch.randn(N, generator=g, device=dev)
    dtype = torch.float16 if epi in (EPI_BIAS_F16, EPI_BIAS_GELU_F16) else torch.float32
    x0 = torch.randn(M, N, generator=g, device=dev) if epi == EPI_BIAS_RESID_F32 else None
    outs = []
    for schedule in (0, 1):
        buf = torch.full((M + GUARD, N), float("nan"), dtype=dtype, device=dev)
        buf[M:] = SENT[dtype]
        if x0 is not None:
            buf[:M] = x0
        _l.check(lib.dss_debug_gemm_schedule(A.data_ptr(), Wt.data_ptr(), bias.data_ptr(), buf.data_ptr(), M, N, K, epi,
                                             schedule, _l.stream_ptr()), "gemm_schedule")
        torch.cuda.synchronize()
        assert torch.equal(buf[M:], torch.full_like(buf[M:], SENT[dtype])), f"schedule {schedule} wrote a guard row"
        outs.append(buf[:M])
    coop, pp = outs
    assert not torch.isnan(coop).any(), "the cooperative schedule left elements unwritten"
    if not torch.equal(coop, pp):
        bad = ~(coop == pp)
        idx = bad.nonzero()[:6].tolist()
        diff = (coop.float() - pp.float()).abs().nan_to_num(float("inf")).max().item()
        raise AssertionError(f"{EPI_NAME[epi]} M={M} N={N} K={K}: {int(bad.sum())} of {bad.numel()} elements differ "
                             f"(max |diff| {diff:.3g}), first at {idx}")
    # and the result is the product (guards against two schedules agreeing on something else)
    ref = torch.addmm(bias.double(), A[:256].double(), Wt.double().T)
    if x0 is not None:
        ref += x0[:256].double()
    if epi == EPI_BIAS_GELU_F16:
        ref = torch.nn.functional.gelu(ref)
    assert torch.allclose(pp[:256].double(), ref, rtol=2e-3, atol=2e-3)


BENCH = [("qkv", EPI_BIAS_F16, 1152, 384), ("fc1", EPI_BIAS_GELU_F16, 1536, 384),
         ("proj", EPI_BIAS_RESID_F32, 384, 384), ("fc2", EPI_BIAS_RESID_F32, 384, 1536)]


@pytest.mark.parametrize("name,epi,N,K", BENCH, ids=[b[0] for b in BENCH])
def test_schedules_agree_bench_shapes(cuda, name, epi, N, K):
    _run(cuda, epi, BENCH_M, N, K, seed=N + K + epi)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("M", [128, 129, 8 * 901])
@pytest.mark.parametrize("epi", list(EPI_NAME), ids=lambda e: EPI_NAME[e])
def test_schedules_agree_rows(cuda, epi, M):
    _run(cuda, epi, M, 384, 384, seed=M + epi)


@pytest.mark.parametrize("epi", list(EPI_NAME), ids=lambda e: EPI_NAME[e])
def test_schedules_agree_odd_items_per_pair(cuda, epi):
    # one row pair per CTA pair and three 128-wide n-tiles: every CTA pair runs 3 items, its group 0 two of them
    pairs = load_pkg("_lib").load().dss_device_sm_count() // 2
    _run(cuda, epi, pairs * 256, 384, 384, seed=3 + epi)


@pytest.mark.parametrize("M,N", [(128, 128), (1000, 384), (2 * 901, 160)])
def test_schedules_agree_fewer_items_than_pairs(cuda, M, N):
    # 1, 12 and 16 work items: CTA pairs with a single item (their group 1 idle)
    for epi in EPI_NAME:
        _run(cuda, epi, M, N, 384, seed=M + N + epi)


@pytest.mark.parametrize("K", [8, 72, 384, 1536])
@pytest.mark.parametrize("epi", list(EPI_NAME), ids=lambda e: EPI_NAME[e])
def test_schedules_agree_k(cuda, epi, K):
    _run(cuda, epi, 8 * 901, 640, K, seed=K + epi)


@pytest.mark.parametrize("N", [96, 160, 1184])
@pytest.mark.parametrize("epi", list(EPI_NAME), ids=lambda e: EPI_NAME[e])
def test_schedules_agree_partial_n_tile(cuda, epi, N):
    # the last 128-wide n-tile holds 96 / 32 / 32 columns (the cooperative schedule runs 128-wide tiles here too)
    _run(cuda, epi, 4 * 901, N, 384, seed=N + epi)
