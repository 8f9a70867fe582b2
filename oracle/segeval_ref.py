"""ORACLE (test infrastructure, not product): numpy restatement of the reference's segmentation evaluation.

  semantic: dataset/voc.py _resize_pseudolabel (cv2), eval.py evaluate + eval_utils.get_iou / hungarian_match /
            majority_vote, computed from a full 256 x 256 confusion (np.bincount) of the valid pixels;
  object:   main.py evaluate_predictions' two-step cv2 downsample and centre crops, metrics.compute_accuracy /
            compute_iou, metrics.mean.

The fixtures under tests/golden/ref_semeval_*.npz and ref_objseg_*.npz hold the reference's own results on seeded
synthetic trees (oracle/make_segeval_golden.py); the CPU tests check this restatement against them, the GPU tests
check the kernel's counts against ``semantic_counts`` / ``object_counts`` here."""
from __future__ import annotations

import cv2
import numpy as np
from scipy.optimize import linear_sum_assignment


def resize_pseudolabel(pseudolabel: np.ndarray, H: int, W: int) -> np.ndarray:
    if pseudolabel.shape[0] in (H // 16, H // 8, 2 * (H // 16)):
        return cv2.resize(pseudolabel, dsize=(W, H), interpolation=cv2.INTER_NEAREST)
    return pseudolabel


def center_crop(x: np.ndarray, S: int) -> np.ndarray:
    top, left = int(round((x.shape[0] - S) / 2.0)), int(round((x.shape[1] - S) / 2.0))
    return x[top:top + S, left:left + S]


def object_prepare(preds: np.ndarray, mask_plane: np.ndarray, downsample, crop: bool):
    """(prediction, target) as compute_metrics sees them: target = R plane >= 128, centre-cropped if crop; prediction
    (already {0, 1}; any dtype cv2 resizes, so that an index map can trace the gather) resized and cropped as
    main.py:88-100."""
    target = mask_plane >= 128
    if crop:
        target = center_crop(target, min(target.shape))
    preds = np.array(preds)
    if downsample is not None:
        H, W = target.shape
        Hp, Wp = preds.shape[0] * downsample, preds.shape[1] * downsample
        preds = cv2.resize(preds, dsize=(max(Wp, W), max(Hp, H)), interpolation=cv2.INTER_NEAREST)
        preds[:Hp, :Wp] = cv2.resize(preds, dsize=(Wp, Hp), interpolation=cv2.INTER_NEAREST)
    if crop:
        preds = center_crop(preds, min(preds.shape))
    return preds, target


def object_counts(preds: np.ndarray, target: np.ndarray) -> np.ndarray:
    p, t = preds.astype(bool), target.astype(bool)
    return np.array([np.sum(p & t), np.sum(p & ~t), np.sum(~p & t), np.sum(~p & ~t)], dtype=np.int64)


def object_image_metrics(preds: np.ndarray, target: np.ndarray):
    """compute_accuracy and compute_iou on numpy: fp32 mean of equality, fp32 intersection / union, NaN -> 0."""
    p, t = preds.astype(bool), target.astype(bool)
    acc = float(np.float32(np.sum(p == t, dtype=np.int64)) / np.float32(p.size))
    inter, union = np.sum(p & (p == t)), np.sum(p | t)
    iou = float(np.float32(inter) / np.float32(union)) if union else 0
    return acc, iou


def mean(x):
    return sum(x) / len(x)


def confusion(pairs) -> np.ndarray:
    """[256, 256] int64: valid pixels (target != 255) per (prediction value, target value) over (pred, target) pairs."""
    M = np.zeros(256 * 256, dtype=np.int64)
    for p, t in pairs:
        valid = t != 255
        M += np.bincount(p[valid].astype(np.int64) * 256 + t[valid], minlength=256 * 256)
    return M.reshape(256, 256)


def semantic_counts(pairs, n_classes: int) -> np.ndarray:
    """The kernel's layout: [256, n_classes + 1], targets >= n_classes (except 255) folded into the last bin."""
    M = confusion(pairs)
    return np.concatenate([M[:, :n_classes], M[:, n_classes:].sum(1, keepdims=True)], axis=1)


VOC_SHAPES = [(500, 375), (375, 500), (333, 500), (500, 333), (500, 500), (281, 500), (366, 500), (500, 400)]


def synthetic_voc_tree(root, n: int = 1449, seed: int = 0, n_clusters: int = 21):
    """A seeded VOC-val-shaped tree under root (VOCdevkit/VOC2012 with JPEGImages, SegmentationClass and the val
    split, and a directory of patch-resolution pseudo-labels at (H // 16, W // 16)), written with PIL. Returns
    (VOC root, segments dir, confusion [256, 256] of the pairs after the reference's resize)."""
    from pathlib import Path
    from PIL import Image
    rng = np.random.default_rng(seed)
    voc = Path(root) / "VOCdevkit" / "VOC2012"
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation"):
        (voc / d).mkdir(parents=True, exist_ok=True)
    seg_dir = Path(root) / "segments"
    seg_dir.mkdir(parents=True, exist_ok=True)
    stems = [f"2010_{i:06d}" for i in range(n)]
    M = np.zeros((256, 256), dtype=np.int64)
    for i, stem in enumerate(stems):
        H, W = VOC_SHAPES[int(rng.integers(len(VOC_SHAPES)))]
        t = np.zeros((H, W), dtype=np.uint8)
        for _ in range(int(rng.integers(1, 4))):
            h, w = int(rng.integers(H // 6, H // 2)), int(rng.integers(W // 6, W // 2))
            y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
            t[max(0, y - 3):y + h + 3, max(0, x - 3):x + w + 3] = 255
            t[y:y + h, x:x + w] = rng.integers(1, 21)
        p = t[8::16, 8::16][:H // 16, :W // 16].astype(np.int64) % n_clusters
        p = np.where(rng.random(p.shape) < 0.15, rng.integers(0, n_clusters, p.shape), p).astype(np.uint8)
        Image.fromarray(np.full((H, W, 3), 128, dtype=np.uint8)).save(voc / "JPEGImages" / f"{stem}.jpg")
        Image.fromarray(t).save(voc / "SegmentationClass" / f"{stem}.png")
        Image.fromarray(p).save(seg_dir / f"{i:05d}.png")
        M += confusion([(resize_pseudolabel(p, H, W), t)])
    (voc / "ImageSets" / "Segmentation" / "val.txt").write_text("".join(f"{s}\n" for s in stems))
    return Path(root), seg_dir, M


def semantic_eval(M: np.ndarray, n_clusters: int, n_classes: int):
    """evaluate() from the confusion M [256, 256]: (eval_result, match, printed lines)."""
    lines = []
    num_elems = int(M.sum())
    rows, cols = M.sum(1), M.sum(0)

    def get_iou(c1, c2):
        tp = int(M[c1, c2]) if c1 < 256 else 0
        fp = int(cols[c2]) - tp
        fn = (int(rows[c1]) if c1 < 256 else 0) - tp
        return float(tp) / max(float(tp + fp + fn), 1e-8)

    if n_clusters == n_classes:
        lines += ["Using hungarian algorithm for matching", "Using iou as metric"]
        res = np.array([get_iou(c1, c2) for c2 in range(n_classes) for c1 in range(n_classes)])
        res = res.reshape((n_classes, n_classes)).T
        m = np.array(list(zip(*linear_sum_assignment(num_elems - res))))
        match = [(out_c, gt_c) for out_c, gt_c in m]
    else:
        lines += ["Using majority voting for matching"]
        res = np.array([get_iou(c1, c2) for c2 in range(n_classes) for c1 in range(n_clusters)])
        res = np.argmax(res.reshape((n_classes, n_clusters)).T, axis=1)
        match = np.array(list(zip(range(n_clusters), res)))
    lines.append(f"Optimal matching: {match}")
    remap = np.zeros(256, dtype=np.int64)
    for pred_i, target_i in match:
        if int(pred_i) < 256:
            remap[int(pred_i)] = int(target_i)
    jac = []
    for i in range(n_classes):
        gt_i = np.zeros(256, dtype=bool)
        gt_i[i] = True
        pred_i = remap == i
        tp = int(M[np.ix_(pred_i, gt_i)].sum())
        fp = int(M[np.ix_(pred_i, ~gt_i)].sum())
        fn = int(M[np.ix_(~pred_i, gt_i)].sum())
        jac.append(float(tp) / max(float(tp + fp + fn), 1e-8))
    result = {"jaccards_all_categs": jac, "mIoU": np.mean(jac)}
    lines += ["Evaluation of semantic segmentation ", "mIoU is %.2f" % (100 * result["mIoU"]), str(result)]
    return result, match, lines
