"""Segmentation-evaluation probe: 1449 seeded VOC-val-shaped pairs (oracle.segeval_ref.synthetic_voc_tree) through

  * the counts kernel alone (CUDA events, warmed up; inputs already on the device): time, pixels/s, bytes addressed;
  * the file-based command (semantic_main): wall time, with the reader threads' decode time measured alone, the
    host->device copy time (pinned, CUDA events) and the kernel time;
  * the reference's host route on the same arrays, restated: the float32 concatenation of the valid pixels and
    get_iou passes (three full numpy passes each) in one process; 21 of the 441 passes are timed and scaled.

    python tools/segeval_probe.py [--out results/segeval_probe.json]
"""
import argparse
import importlib
import io
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
se = importlib.import_module("deep-spectral-segmentation_b200.segeval")
from oracle import segeval_ref  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=1449)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu, "pairs": args.n}
    with tempfile.TemporaryDirectory() as d:
        root, seg_dir, M = segeval_ref.synthetic_voc_tree(d, args.n, seed=3)
        images, targets, segments, _ = se.voc_pairs(str(root), "2012", "val", str(seg_dir))

        t0 = time.perf_counter()
        maps = se._map_threads(lambda i: (se._read_u8(segments[i]), se._read_u8(targets[i])), range(args.n))
        res["reader_s"] = time.perf_counter() - t0
        items = [(p, t, se.semantic_gather(p.shape, t.shape, t.shape)) for p, t in maps]
        pix = sum(t.size for _, t, _ in items)
        res["pixels"] = pix
        # bytes addressed: target bytes, one prediction byte and one column-table int32 per pixel, the tables, counts
        res["bytes_addressed"] = int(pix * (1 + 1 + 4) + sum(g.table().nbytes for _, _, g in items) + 256 * 22 * 8)

        # kernel alone on device-resident inputs
        preds = torch.from_numpy(np.concatenate([p.reshape(-1) for p, _, _ in items])).to(dev)
        tgts = torch.from_numpy(np.concatenate([t.reshape(-1) for _, t, _ in items])).to(dev)
        desc = np.zeros((len(items), 13), dtype=np.int64)
        po = to = tab = 0
        for b, (p, t, g) in enumerate(items):
            desc[b] = (po, *p.shape, to, *t.shape, 0, 0, g.h, g.w, 0, 0, tab)
            po, to, tab = po + p.size, to + t.size, tab + 2 * (g.h + g.w)
        tables = np.concatenate([g.table() for _, _, g in items])
        lib = se._lib.load()
        counts = torch.zeros(256, 22, dtype=torch.int64, device=dev)
        ws = torch.empty(int(lib.dss_segeval_workspace_bytes(len(items), len(tables))), dtype=torch.uint8, device=dev)

        def run():
            se._lib.check(lib.dss_segeval_counts(preds.data_ptr(), preds.numel(), tgts.data_ptr(), tgts.numel(),
                                                 desc.ctypes.data, len(items), tables.ctypes.data, len(tables), 0, 21,
                                                 counts.data_ptr(), ws.data_ptr(), ws.numel(),
                                                 se._lib.stream_ptr(dev)))
        for _ in range(3):
            run()
        reps = 20
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        counts.zero_()
        e0.record()
        for _ in range(reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        want = np.concatenate([M[:, :21], M[:, 21:].sum(1, keepdims=True)], 1)
        assert np.array_equal(counts.cpu().numpy(), reps * want), "kernel counts differ from the oracle"
        res["kernel_ms"] = ms
        res["kernel_pixels_per_s"] = pix / (ms / 1e3)
        res["kernel_bytes_per_s"] = res["bytes_addressed"] / (ms / 1e3)

        # host->device copy of the same bytes from pinned memory
        hp = torch.cat([preds.cpu(), tgts.cpu()]).pin_memory()
        hd = torch.empty_like(hp, device=dev)
        hd.copy_(hp, non_blocking=True)
        e0.record()
        hd.copy_(hp, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        res["copy_ms"] = e0.elapsed_time(e1)
        res["copy_bytes"] = hp.numel()

        # the file-based command end to end
        se.semantic_main([f"segments_dir={seg_dir}", f"data.val_kwargs.root={root}"], out=io.StringIO())  # warm
        t0 = time.perf_counter()
        se.semantic_main([f"segments_dir={seg_dir}", f"data.val_kwargs.root={root}"], out=io.StringIO())
        res["command_s"] = time.perf_counter() - t0

        # the reference's host route (restated): float32 concatenation, then get_iou passes in one process
        t0 = time.perf_counter()
        all_preds = np.zeros(args.n * 500 * 500, dtype=np.float32)
        all_gt = np.zeros(args.n * 500 * 500, dtype=np.float32)
        off = 0
        for p, t, g in items:
            valid = t != 255
            n = int(valid.sum())
            all_gt[off:off + n] = t[valid]
            all_preds[off:off + n] = p[np.ix_(g.rows_out, g.cols_out)][valid]
            off += n
        all_preds, all_gt = all_preds[:off], all_gt[:off]
        res["ref_concat_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        for c1 in range(21):
            a, b = all_preds == c1, all_gt == 0
            int(np.sum(a & b)), int(np.sum(~a & b)), int(np.sum(a & ~b))
        res["ref_21_get_iou_s"] = time.perf_counter() - t0
        res["ref_441_get_iou_s_scaled"] = res["ref_21_get_iou_s"] * 21
    print(json.dumps(res, indent=1))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
