"""LOST and DINO-seg throughput on ragged batches against the per-size grouping, on one GPU.

    python tools/ragged_localize_probe.py [--out DIR] [--reps 3] [--batch 16]

ViT-S/16, fp16 mode, seeded weights, on the 512 long-tailed image sizes of tools/ragged_probe.py (70 %
synth.VOC_SHAPES, 30 % a tail with one side 500). Per-size: the images grouped by size into batches of up to --batch
(what object-localization/main.py did before: forward_last + lost_boxes / dinoseg_boxes per batch); ragged: batches of
--batch in list order (forward_last_ragged + lost_boxes_ragged / dinoseg_boxes_ragged). Images/s from CUDA events
around the whole route, boxes included, after a warm-up; the two variants alternated; and whether their boxes, seeds
and status are bitwise equal. Prints the card's name and power limit and one JSON line (also DIR/ragged_localize_probe.json
with --out)."""
from __future__ import annotations

import argparse
import importlib
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import ragged_probe  # noqa: E402

PKG = "deep-spectral-segmentation_b200"
vit = importlib.import_module(PKG + ".vit")
loc = importlib.import_module(PKG + ".localize")
P = 16


def per_size_batches(shapes, bs):
    """The former grouping: images keyed by size, a group flushed when it reaches bs, the rest at the end."""
    pending, out = {}, []
    for j, s in enumerate(shapes):
        pending.setdefault(s, []).append(j)
        if len(pending[s]) >= bs:
            out.append(pending.pop(s))
    return out + list(pending.values())


def run_per_size(model, ims, batches, method):
    res = {}
    for idx in batches:
        x = torch.stack([ims[j] for j in idx])
        H, W = ims[idx[0]].shape[:2]
        grid = (-(-H // P), -(-W // P))
        if method == "lost":
            f, _ = model.forward_last(x, "k", pad=True)
            b, s, st = loc.lost_boxes(f, grid, (H, W), P, 100)
        else:
            _, a = model.forward_last(x, "k", pad=True, feats=False, cls_attn=True)
            b, st = loc.dinoseg_boxes(a, grid, P, 4)
            s = st
        for t, j in enumerate(idx):
            res[j] = (b[t].tolist(), int(s[t]), int(st[t]))
    return res


def run_ragged(model, packed, dims, offsets, bs, method):
    res = {}
    n = dims.shape[0]
    for s0 in range(0, n, bs):
        s1 = min(n, s0 + bs)
        d = dims[s0:s1]
        x = packed[offsets[s0]:offsets[s1]]
        if method == "lost":
            f, _, grids = model.forward_last_ragged(x, d, "k", pad=True)
            b, s, st = loc.lost_boxes_ragged(f, [g[1:] for g in grids], d.tolist(), P, 100)
        else:
            _, a, grids = model.forward_last_ragged(x, d, "k", pad=True, feats=False, cls_attn=True)
            b, st = loc.dinoseg_boxes_ragged(a, [g[1:] for g in grids], P, 4)
            s = st
        for t in range(s1 - s0):
            res[s0 + t] = (b[t].tolist(), int(s[t]), int(st[t]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    card = ragged_probe.card()
    print("card:", card)
    model = vit.get_model("dino_vits16", seed=0, device="cuda")[0]
    shapes = ragged_probe.image_shapes(512)
    g = torch.Generator().manual_seed(1)
    ims = [torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g).cuda() for H, W in shapes]
    packed, dims = vit.pack_images(ims)
    offsets = np.concatenate([[0], np.cumsum([H * W for H, W in shapes])])
    batches = per_size_batches(shapes, a.batch)
    out = {"card": card, "images": len(shapes), "distinct_shapes": len(set(shapes)), "batch": a.batch,
           "per_size_forwards": len(batches), "ragged_forwards": -(-len(shapes) // a.batch)}
    for method in ("lost", "dinoseg"):
        per_size = lambda: run_per_size(model, ims, batches, method)
        ragged = lambda: run_ragged(model, packed, dims, offsets, a.batch, method)
        og, _ = ragged_probe.timed(per_size)   # warm-up: every shape
        orr, _ = ragged_probe.timed(ragged)
        tg, tr = [], []
        for _ in range(a.reps):
            tg.append(ragged_probe.timed(per_size)[1])
            tr.append(ragged_probe.timed(ragged)[1])
        n = len(shapes)
        out[method] = {"per_size_images_per_s": [round(n / t, 1) for t in tg],
                       "ragged_images_per_s": [round(n / t, 1) for t in tr],
                       "bitwise_equal": all(og[j] == orr[j] for j in range(n)),
                       "failed_images": sum(1 for j in range(n) if orr[j][2] != 0)}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "ragged_localize_probe.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
