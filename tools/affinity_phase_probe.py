"""Where the time inside a tile of the affinity GEMM goes, at the benchmark's step (B = 264 images, N = 900 patches,
d = 384, normalised features, degree on): dss_debug_affinity_trace, %globaltimer stamps.

It prints the card's name, power limit and clocks (nvidia-smi, read in the same run), the CUDA-event time of the whole
dss_affinity call and, from torch.profiler, of each kernel it launches, then from one traced launch the mean per-tile
split: waiting for the first operand slab, wgmma main loop, epilogue, and the producer warp's wait on empty ring
slots per tile. The split is given for all tiles and by tile kind: strictly upper tiles, diagonal tiles, tiles of the
image's last column tile (4 real columns at N = 900) and the odd CTA's discarded tiles below the diagonal. Per CTA it
gives the span (first tile start to last epilogue issued) and the share of it in which the CTA's consumer groups were
not in their main loop ("tensor idle": operand waits plus epilogues, which the cooperative schedule does not overlap).

    python tools/affinity_phase_probe.py [--out DIR]
"""
import argparse
import importlib
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_lib = importlib.import_module("deep-spectral-segmentation_b200._lib")

B, N, D = 264, 900, 384
NORMALIZE = 1


def cdiv(a, b):
    return (a + b - 1) // b


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def tile_kinds(clusters, tmax):
    """[2 * clusters, tmax] kind of the j-th tile of each CTA: 0 upper, 1 diagonal, 2 last column tile, 3 discarded"""
    tiles = cdiv(N, 128)
    order = [(p, j) for p in range(cdiv(tiles, 2)) for j in range(2 * p, tiles)]
    kinds = torch.full((2 * clusters, tmax), -1, dtype=torch.int64)
    for c in range(2 * clusters):
        cid, rank = c >> 1, c & 1
        for j in range(tmax):
            t = cid + j * clusters
            if t >= B * len(order):
                break
            p, n = order[t % len(order)]
            m = 2 * p + rank
            kinds[c, j] = 3 if m > n else 2 if n == tiles - 1 else 1 if m == n else 0
    return kinds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="", help="directory for affinity_phase_probe.json")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    lib = _lib.load()
    dev = torch.device("cuda:0")
    res = {"card": card(), "device": torch.cuda.get_device_name(dev), "sms": int(lib.dss_device_sm_count()),
           "B": B, "N": N, "d": D}
    print(res["card"], flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    f = torch.randn(B, N, D, generator=g, device=dev)
    ldw = N
    W = torch.empty(B, N, ldw, device=dev)
    deg = torch.empty(B, N, device=dev)
    need = int(lib.dss_affinity_workspace_bytes(B, N, D))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr()

    def run():
        _lib.check(lib.dss_affinity(f.data_ptr(), B, N, D, NORMALIZE, None, 0.0, W.data_ptr(), ldw, deg.data_ptr(),
                                    ws.data_ptr(), need, st), "dss_affinity")

    for _ in range(3):
        run()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.reps):
        run()
    ev[1].record()
    torch.cuda.synchronize()
    res["affinity_call_ms"] = ev[0].elapsed_time(ev[1]) / args.reps

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            run()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.count > 0:
            kernels[e.key[:60]] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / args.reps / 1e3
    res["kernel_ms"] = kernels

    tiles = cdiv(N, 128)
    items = B * sum(max(tiles - 2 * p, 0) for p in range(cdiv(tiles, 2)))
    clusters = min(items, res["sms"] // 2)
    tmax = cdiv(items, clusters)
    stride = 4 + 8 * tmax
    trace = torch.zeros(2 * clusters * stride, dtype=torch.int64, device=dev)
    _lib.check(lib.dss_debug_affinity_trace(f.data_ptr(), B, N, D, NORMALIZE, None, 0.0, W.data_ptr(), ldw,
                                            deg.data_ptr(), ws.data_ptr(), need, trace.data_ptr(), trace.numel() * 8,
                                            st), "debug_affinity_trace")
    torch.cuda.synchronize()
    tr = trace.view(2 * clusters, stride).cpu().double()
    rec = tr[:, 4:].view(2 * clusters, 2, tmax, 4)
    valid = rec[..., 0] > 0
    t0, t1, t2, t3 = (rec[..., i] for i in range(4))
    kinds = tile_kinds(clusters, tmax)[:, None, :].expand(-1, 2, -1)

    def split(mask):
        w, m, e = (t1 - t0)[mask], (t2 - t1)[mask], (t3 - t2)[mask]
        return {"tiles": int(mask.sum()) // 2, "operand_wait_us": float(w.mean()) / 1e3,
                "mainloop_us": float(m.mean()) / 1e3, "epilogue_us": float(e.mean()) / 1e3,
                "tile_us": float((t3 - t0)[mask].mean()) / 1e3}

    res["per_tile"] = {"all": split(valid)}
    for k, name in enumerate(["upper", "diagonal", "last_column", "discarded"]):
        res["per_tile"][name] = split(valid & (kinds == k))
    big = torch.tensor(float("inf"), dtype=torch.float64)
    span = torch.where(valid, t3, -big).amax(dim=(1, 2)) - torch.where(valid, t0, big).amin(dim=(1, 2))
    main_cta = ((t2 - t1) * valid)[:, 0].sum(dim=1)   # both groups run the same tile at once: count group 0
    tiles_cta = valid[:, 0].sum(dim=1)
    res["producer_wait_us_per_tile"] = float(tr[:, 0].sum() / tiles_cta.sum()) / 1e3
    res["cta_span_us_mean"] = float(span.mean()) / 1e3
    res["cta_span_us_max"] = float(span.max()) / 1e3
    res["tensor_idle_share"] = float((1 - main_cta / span).mean())

    print(f"{res['device']}, {res['sms']} SMs; B = {B}, N = {N}, d = {D}: dss_affinity {res['affinity_call_ms']:.3f} ms")
    for k, v in kernels.items():
        print(f"  kernel {v:7.3f} ms  {k}")
    for k, v in res["per_tile"].items():
        print(f"  {k:11s} {v['tiles']:5d} tiles: {v['tile_us']:6.2f} us = operands {v['operand_wait_us']:5.2f} + main "
              f"{v['mainloop_us']:5.2f} + epilogue {v['epilogue_us']:5.2f}")
    print(f"  producer empty-wait {res['producer_wait_us_per_tile']:.2f} us per tile; CTA span {res['cta_span_us_mean']:.1f}"
          f" us (max {res['cta_span_us_max']:.1f}), tensor idle {100 * res['tensor_idle_share']:.1f} %", flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "affinity_phase_probe.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
