"""ViT throughput of ragged batches against the per-shape grouping, on one GPU.

    python tools/ragged_probe.py [--out DIR] [--reps 3]

ViT-S/16, fp16 mode, seeded weights, batch_size 64, on two inputs:
  (a) 512 images from a long-tailed size table: synth.VOC_SHAPES plus a tail of sizes with a maximum side of 500;
  (b) about 2000 box crops with the shapes extract_bboxes produces: boxes on the patch grid of 375 x 500 / 500 x 375
      images, multiples of the patch size clipped at the image border, from synthetic multi-region label maps.
For each: forward_k (a) or forward_cls (b) over per-shape batches of up to 64 (what the commands did before) and over
ragged batches of 64 in list order; ViT images/s from CUDA events after a warm-up, the two variants alternated; the
number of ViT forwards; the number of distinct shapes; and whether the two variants' outputs are bitwise equal. Prints
the card's name and power limit and one JSON line (written to DIR/ragged_probe.json with --out)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import importlib  # noqa: E402

PKG = "deep-spectral-segmentation_b200"
vit = importlib.import_module(PKG + ".vit")
synth = importlib.import_module(PKG + ".synth")

BS, P = 64, 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def image_shapes(n, seed=0):
    """70 % synth.VOC_SHAPES, 30 % a tail: one side 500, the other uniform in [160, 500]."""
    rng = np.random.default_rng(seed)
    voc = synth.voc_shapes(n, seed)
    out = []
    for i in range(n):
        if rng.random() < 0.7:
            out.append(voc[i])
        else:
            s = int(rng.integers(160, 501))
            out.append((500, s) if rng.random() < 0.5 else (s, 500))
    return out


def crop_shapes(n, seed=0):
    """Box crops as extract_bboxes makes them: each synthetic label map (a 375 x 500 or 500 x 375 image, its patch grid
    cut into 2..6 rectangular regions) gives one box per region, in patch units, scaled to pixels and clipped."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        H, W = (375, 500) if rng.random() < 0.7 else (500, 375)
        hp, wp = -(-H // P), -(-W // P)
        for _ in range(int(rng.integers(2, 7))):
            y0, x0 = int(rng.integers(0, hp)), int(rng.integers(0, wp))
            y1, x1 = int(rng.integers(y0 + 1, hp + 1)), int(rng.integers(x0 + 1, wp + 1))
            out.append((min(y1 * P, H) - y0 * P, min(x1 * P, W) - x0 * P))
    return [s for s in out[:n] if s[0] >= P and s[1] >= P]


def grouped_batches(shapes):
    groups = defaultdict(list)
    for i, s in enumerate(shapes):
        groups[s].append(i)
    return [idx[j:j + BS] for idx in groups.values() for j in range(0, len(idx), BS)]


def run_grouped(model, ims, batches, cls):
    outs = {}
    for idx in batches:
        x = torch.stack([ims[i] for i in idx])
        y = model.forward_cls(x) if cls else model.forward_k(x)
        for j, i in enumerate(idx):
            outs[i] = y[j]
    return outs


def run_ragged(model, packed, dims, offsets, cls):
    outs = {}
    n = dims.shape[0]
    for s in range(0, n, BS):
        e = min(s + BS, n)
        x = packed[offsets[s]:offsets[e]]
        if cls:
            y, _ = model.forward_cls_ragged(x, dims[s:e])
            for j in range(e - s):
                outs[s + j] = y[j]
        else:
            y, rows = model.forward_k_ragged(x, dims[s:e])
            for j, (r0, r1) in enumerate(rows):
                outs[s + j] = y[r0:r1]
    return outs


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3


def measure(model, shapes, cls, reps):
    g = torch.Generator().manual_seed(1)
    ims = [torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g).cuda() for H, W in shapes]
    packed, dims = vit.pack_images(ims)
    offsets = np.concatenate([[0], np.cumsum([H * W for H, W in shapes])])
    batches = grouped_batches(shapes)
    grouped = lambda: run_grouped(model, ims, batches, cls)
    ragged = lambda: run_ragged(model, packed, dims, offsets, cls)
    og, _ = timed(grouped)   # warm-up: every shape
    orr, _ = timed(ragged)
    tg, tr = [], []
    for _ in range(reps):
        tg.append(timed(grouped)[1])
        tr.append(timed(ragged)[1])
    equal = all(torch.equal(og[i], orr[i]) for i in range(len(shapes)))
    n = len(shapes)
    return {"images": n, "distinct_shapes": len(set(shapes)), "grouped_forwards": len(batches),
            "ragged_forwards": -(-n // BS), "grouped_images_per_s": [round(n / t, 1) for t in tg],
            "ragged_images_per_s": [round(n / t, 1) for t in tr], "bitwise_equal": equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    model = vit.get_model("dino_vits16", seed=0, device="cuda")[0]
    res = {"card": card(), "batch_size": BS,
           "images_forward_k": measure(model, image_shapes(512), False, a.reps),
           "box_crops_forward_cls": measure(model, crop_shapes(2000), True, a.reps)}
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "ragged_probe.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
