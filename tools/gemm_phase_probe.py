"""Where the time inside a GEMM tile goes, for the four ViT-S/16 GEMM classes of one benchmark step (M = 264 * 901 rows),
under the cooperative and the ping-pong schedule (dss_debug_gemm_trace / dss_debug_gemm_schedule).

Per class and schedule it prints the CUDA-event time of the untraced kernel and, from one traced launch, the mean per-tile
split (waiting for the first operand slab, wgmma main loop, epilogue), the producer warp's wait on empty ring slots, and
the per-CTA timeline: span (first tile start to last epilogue issued) and the share of it in which no consumer group
of the CTA was in its main loop ("tensor idle"). Under the cooperative schedule that idle share is the epilogue plus
the operand waits; under the ping-pong schedule a group's epilogue runs while the other group's main loop runs.

    python tools/gemm_phase_probe.py [--out DIR]
"""
import argparse
import importlib
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_lib = importlib.import_module("deep-spectral-segmentation_b200._lib")

M = 264 * 901
CLASSES = [   # name, epilogue, N, K
    ("qkv", _lib.EPI_BIAS_F16, 1152, 384),
    ("fc1", _lib.EPI_BIAS_GELU_F16, 1536, 384),
    ("proj", _lib.EPI_BIAS_RESID_F32, 384, 384),
    ("fc2", _lib.EPI_BIAS_RESID_F32, 384, 1536),
]
SCHEDULES = {0: "cooperative", 1: "ping-pong"}


def cdiv(a, b):
    return (a + b - 1) // b


def tile_n(schedule, N):
    if schedule == 1:
        return 128
    return 256 if N % 256 == 0 else (192 if N % 192 == 0 else 128)


def probe(lib, dev, name, epi, N, K, schedule, reps=10):
    g = torch.Generator(device=dev).manual_seed(1000 + N + K + epi)
    A = torch.randn(M, K, generator=g, device=dev).half()
    Wt = (torch.randn(N, K, generator=g, device=dev) * K ** -0.5).half()
    bias = torch.randn(N, generator=g, device=dev)
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if epi == _lib.EPI_BIAS_RESID_F32 else torch.float16)
    st = _lib.stream_ptr()

    def run():
        _lib.check(lib.dss_debug_gemm_schedule(A.data_ptr(), Wt.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K,
                                               epi, schedule, st), "gemm_schedule")

    for _ in range(3):
        run()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        run()
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / reps

    bn = tile_n(schedule, N)
    items = cdiv(cdiv(M, 128), 2) * cdiv(N, bn)
    clusters = min(items, lib.dss_device_sm_count() // 2)
    tmax = cdiv(items, clusters)
    stride = 4 + 8 * tmax
    trace = torch.zeros(2 * clusters * stride, dtype=torch.int64, device=dev)
    _lib.check(lib.dss_debug_gemm_trace(A.data_ptr(), Wt.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K, epi,
                                        schedule, trace.data_ptr(), trace.numel() * 8, st), "gemm_trace")
    torch.cuda.synchronize()
    tr = trace.view(2 * clusters, stride).cpu().double()
    prod_wait = tr[:, 0]
    rec = tr[:, 4:].view(2 * clusters, 2, tmax, 4)
    valid = rec[..., 0] > 0
    t0, t1, t2, t3 = (rec[..., i] for i in range(4))
    wait, main, epi_t = (t1 - t0)[valid], (t2 - t1)[valid], (t3 - t2)[valid]
    tile = (t3 - t0)[valid]
    big = torch.tensor(float("inf"), dtype=torch.float64)
    start = torch.where(valid, t0, big).amin(dim=(1, 2))
    end = torch.where(valid, t3, -big).amax(dim=(1, 2))
    span = end - start
    # main-loop time of the CTA: the cooperative groups run the same tile at once (count one group), the ping-pong
    # groups take turns (count both)
    main_cta = ((t2 - t1) * valid)[:, 0].sum(dim=1) if schedule == 0 else ((t2 - t1) * valid).sum(dim=(1, 2))
    tiles_cta = valid[:, 0].sum(dim=1) if schedule == 0 else valid.sum(dim=(1, 2))
    res = {
        "class": name, "schedule": SCHEDULES[schedule], "M": M, "N": N, "K": K, "tile": f"128x{bn}",
        "kernel_ms": ms, "tflops": 2.0 * M * N * K / ms / 1e9,
        "tile_us": float(tile.mean()) / 1e3, "operand_wait_us": float(wait.mean()) / 1e3,
        "mainloop_us": float(main.mean()) / 1e3, "epilogue_us": float(epi_t.mean()) / 1e3,
        "epilogue_share": float(epi_t.mean() / tile.mean()),
        "producer_wait_us_per_tile": float(prod_wait.sum() / tiles_cta.sum()) / 1e3,
        "cta_span_us_mean": float(span.mean()) / 1e3, "cta_span_us_max": float(span.max()) / 1e3,
        "cta_span_per_tile_us": float((span / tiles_cta).mean()) / 1e3,
        "tensor_idle_share": float((1 - main_cta / span).mean()),
    }
    print(f"{name:4s} {SCHEDULES[schedule]:11s} 128x{bn:<3d} {ms:7.3f} ms {res['tflops']:6.1f} TFLOP/s | per tile "
          f"{res['tile_us']:6.2f} us: operands {res['operand_wait_us']:5.2f} main {res['mainloop_us']:5.2f} "
          f"epilogue {res['epilogue_us']:5.2f} ({100 * res['epilogue_share']:4.1f} %), producer empty-wait "
          f"{res['producer_wait_us_per_tile']:5.2f} | CTA span {res['cta_span_us_mean']:7.1f} us "
          f"(max {res['cta_span_us_max']:7.1f}), {res['cta_span_per_tile_us']:5.2f} us per tile, tensor idle "
          f"{100 * res['tensor_idle_share']:4.1f} %", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="", help="directory for gemm_phase_probe.json")
    ap.add_argument("--schedules", default="0,1")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    lib = _lib.load()
    dev = torch.device("cuda:0")
    print(f"{torch.cuda.get_device_name(dev)}, {lib.dss_device_sm_count()} SMs, M = {M}")
    rows = [probe(lib, dev, name, epi, N, K, int(s)) for name, epi, N, K in CLASSES for s in args.schedules.split(",")]
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "gemm_phase_probe.json").write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
