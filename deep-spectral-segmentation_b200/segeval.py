"""Segmentation evaluation (the reference's semantic-segmentation/eval.py + eval_utils.py + dataset/voc.py, and
object-segmentation/main.py + metrics.py + dataset.py): mIoU of semantic pseudo-labels with Hungarian or majority-vote
matching, and per-image pixel accuracy and IoU of binary object masks.

Device work: csrc/segeval.cu turns a ragged batch of (prediction, target) label maps into exact integer counts. Every
resize and crop of the reference is a host-built gather table (``crf._nn_index``, the cv2 INTER_NEAREST rule), so the
counts are the reference's pixels exactly. Everything after the counts (IoU matrix, matching, remap, TP / FP / FN,
mIoU, per-image acc / IoU and their means) follows from them on the host, in the reference's own arithmetic.

The commands read PNG label maps on reader threads (images are never decoded: the semantic app reads only JPEG sizes,
the object app only the masks), stage batches through pinned memory, and copy the counts back once per data set
(semantic) or once per batch (binary). Single process, one GPU. See DESIGN.md section 5 for the differences from the
reference."""
from __future__ import annotations

import os
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, io_pipeline
from .crf import _nn_index

MAX_CLASSES = 63          # num_classes + 1 target bins of one CTA's shared-memory histogram (<= 64)
BATCH = 64                # images per kernel call of the commands
VOC_RESIZE_RULE = (16, 8)  # dataset/voc.py:12-19: H // 16, H // 8 and 2 * (H // 16)


# ------------------------------------------------------------------------------------------------ gather tables
class Gather:
    """Where output pixel (y, x) of one image reads: target (top + y, left + x), prediction (rows[y], cols[x]); the
    ``_in`` tables inside the top-left block (y < block_h, x < block_w), the ``_out`` tables elsewhere."""
    __slots__ = ("top", "left", "h", "w", "rows_in", "rows_out", "cols_in", "cols_out", "block_h", "block_w")

    def __init__(self, top, left, rows_in, rows_out, cols_in, cols_out, block_h=0, block_w=0):
        self.top, self.left = int(top), int(left)
        self.h, self.w = len(rows_out), len(cols_out)
        self.rows_in, self.rows_out = np.asarray(rows_in), np.asarray(rows_out)
        self.cols_in, self.cols_out = np.asarray(cols_in), np.asarray(cols_out)
        self.block_h, self.block_w = int(block_h), int(block_w)

    def table(self) -> np.ndarray:
        return np.concatenate([self.rows_in, self.rows_out, self.cols_in, self.cols_out]).astype(np.int32)


def center_crop_offsets(H: int, W: int, S: int) -> Tuple[int, int]:
    """torchvision's center_crop offsets (top, left): int(round(d / 2.0)), Python's banker's rounding."""
    return int(round((H - S) / 2.0)), int(round((W - S) / 2.0))


def semantic_gather(pred_shape, image_shape, target_shape, name: str = "") -> Gather:
    """_resize_pseudolabel (dataset/voc.py:12-19): a nearest resize to the image size when the map's height is H // 16,
    H // 8 or 2 (H // 16), the map itself otherwise. The result must have the target's shape (the reference's boolean
    index fails otherwise)."""
    ph, pw = pred_shape
    H, W = image_shape
    if ph in (H // 16, H // 8, 2 * (H // 16)):
        rows, cols = _nn_index(H, ph), _nn_index(W, pw)
    else:
        rows, cols = np.arange(ph), np.arange(pw)
    if (len(rows), len(cols)) != tuple(target_shape):
        raise ValueError(f"{name}: the pseudo-label of shape {ph} x {pw} becomes {len(rows)} x {len(cols)} for an "
                         f"image of {H} x {W}, but the target is {target_shape[0]} x {target_shape[1]}")
    return Gather(0, 0, rows, rows, cols, cols)


def object_gather(pred_shape, mask_shape, downsample: Optional[int], crop: bool, name: str = "") -> Gather:
    """evaluate_predictions (object-segmentation/main.py:88-100) on a mask of mask_shape (before the data set's centre
    crop): the optional two-step downsample resize -- resize to (H_max, W_max), then the top-left H_pad x W_pad block
    overwritten by a resize of that already-resized map -- and the optional centre crops of the target and the
    prediction."""
    MH, MW = mask_shape
    top, left, H, W = 0, 0, MH, MW
    if crop:
        H = W = min(MH, MW)
        top, left = center_crop_offsets(MH, MW, H)
    ph, pw = pred_shape
    if downsample is not None:
        Hp, Wp = ph * downsample, pw * downsample
        Hm, Wm = max(Hp, H), max(Wp, W)
        r1, c1 = _nn_index(Hm, ph), _nn_index(Wm, pw)
        rin, cin = r1.copy(), c1.copy()
        rin[:Hp], cin[:Wp] = r1[_nn_index(Hp, Hm)], c1[_nn_index(Wp, Wm)]
    else:
        Hp = Wp = 0
        r1, c1 = np.arange(ph), np.arange(pw)
        rin, cin = r1, c1
    ptop, pleft, PH, PW = 0, 0, len(r1), len(c1)
    if crop:
        S = min(PH, PW)
        ptop, pleft = center_crop_offsets(PH, PW, S)
        PH = PW = S
    if (PH, PW) != (H, W):
        hint = (" (full-resolution masks need predictions.downsample=null)" if downsample is not None
                else " (patch-resolution masks need predictions.downsample=<patch size>)")
        raise ValueError(f"{name}: the prediction of shape {ph} x {pw} becomes {PH} x {PW}, but the ground truth is "
                         f"{H} x {W}{hint}")
    return Gather(top, left, rin[ptop:ptop + H], r1[ptop:ptop + H], cin[pleft:pleft + W], c1[pleft:pleft + W],
                  max(0, Hp - ptop), max(0, Wp - pleft))


# ------------------------------------------------------------------------------------------------ device counts
@torch.no_grad()
def _counts(items: Sequence[Tuple[np.ndarray, np.ndarray, Gather]], mode: int, num_classes: int,
            counts: torch.Tensor) -> None:
    """One dss_segeval_counts call; items = (prediction uint8 [ph, pw], target uint8 [th, tw], Gather)."""
    B = len(items)
    desc = np.zeros((B, _lib.SEGEVAL_FIELDS), dtype=np.int64)
    po = to = tab = 0
    for b, (p, t, g) in enumerate(items):
        desc[b] = (po, p.shape[0], p.shape[1], to, t.shape[0], t.shape[1], g.top, g.left, g.h, g.w, g.block_h,
                   g.block_w, tab)
        po, to, tab = po + p.size, to + t.size, tab + 2 * (g.h + g.w)
    tables = np.concatenate([g.table() for _, _, g in items])
    dev = counts.device
    preds = torch.from_numpy(np.concatenate([p.reshape(-1) for p, _, _ in items])).pin_memory().to(dev, non_blocking=True)
    targets = torch.from_numpy(np.concatenate([t.reshape(-1) for _, t, _ in items])).pin_memory().to(dev,
                                                                                                       non_blocking=True)
    lib = _lib.load()
    with torch.cuda.device(dev):
        ws = torch.empty(max(256, int(lib.dss_segeval_workspace_bytes(B, len(tables)))), dtype=torch.uint8, device=dev)
        _lib.check(lib.dss_segeval_counts(preds.data_ptr(), preds.numel(), targets.data_ptr(), targets.numel(),
                                          desc.ctypes.data, B, tables.ctypes.data, len(tables), mode, num_classes,
                                          counts.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)),
                   "dss_segeval_counts")


def semantic_counts(items, n_classes: int, counts: Optional[torch.Tensor] = None, device=None) -> torch.Tensor:
    """Adds the (prediction value, target bin) pixel counts of items = [(prediction, target, Gather)] into counts
    [256, n_classes + 1] int64 on the device (allocated zero if None) and returns it. Target 255 is ignored; bins
    0 .. n_classes - 1 are the classes, bin n_classes every other target value. Call once per batch of a data set."""
    if not 1 <= n_classes <= MAX_CLASSES:
        raise ValueError(f"{n_classes} classes: 1 .. {MAX_CLASSES} are supported")
    if counts is None:
        counts = torch.zeros(256, n_classes + 1, dtype=torch.int64, device=device or torch.device("cuda"))
    _lib.require_cuda(counts, "counts")
    assert counts.dtype == torch.int64 and counts.is_contiguous() and tuple(counts.shape) == (256, n_classes + 1)
    if items:
        _counts(items, _lib.SEGEVAL_SEMANTIC, n_classes, counts)
    return counts


def object_counts(items, device=None) -> np.ndarray:
    """Per-image int64 [B, 4] = {TP, FP, FN, TN} of prediction != 0 against target >= 128 (ToTensor() > 0.5)."""
    out = torch.empty(len(items), 4, dtype=torch.int64, device=device or torch.device("cuda"))
    if items:
        _counts(items, _lib.SEGEVAL_BINARY, 0, out)
    return out.cpu().numpy()


# ------------------------------------------------------------------------------------------------ host arithmetic
def iou_matrix(counts: np.ndarray, n_clusters: int, n_classes: int) -> np.ndarray:
    """get_iou (eval_utils.py:36-46) of every (cluster c1, class c2): float(tp) / max(float(tp + fp + fn), 1e-8), the
    row total of c1 over every valid target value, the column total of c2 over every prediction value 0 .. 255."""
    C = np.asarray(counts, dtype=np.int64)
    Cp = np.zeros((max(n_clusters, 256), C.shape[1]), dtype=np.int64)
    Cp[:256] = C
    tp = Cp[:n_clusters, :n_classes]
    fn = Cp[:n_clusters].sum(1)[:, None] - tp
    fp = C[:, :n_classes].sum(0)[None, :] - tp
    return tp.astype(np.float64) / np.maximum((tp + fp + fn).astype(np.float64), 1e-8)


def match_clusters(counts, n_clusters: int, n_classes: int):
    """hungarian_match (n_clusters == n_classes: scipy's linear_sum_assignment on num_valid_pixels - IoU, a list of
    (cluster, class) numpy int64 pairs) or majority_vote (argmax over classes, first wins on ties: an int64 array
    [n_clusters, 2]) -- the reference's objects, so that they print the same."""
    from scipy.optimize import linear_sum_assignment
    counts = np.asarray(counts, dtype=np.int64)
    if n_clusters == n_classes:
        match = linear_sum_assignment(int(counts.sum()) - iou_matrix(counts, n_clusters, n_classes))
        return [(out_c, gt_c) for out_c, gt_c in np.array(list(zip(*match)))]
    return np.array(list(zip(range(n_clusters), np.argmax(iou_matrix(counts, n_clusters, n_classes), axis=1))))


def semantic_miou(counts, match, n_classes: int) -> dict:
    """Remap (values absent from the match go to class 0), per-class TP / FP / FN and the Jaccard indices
    (eval.py:136-157): {'jaccards_all_categs': [float], 'mIoU': np.mean of them}."""
    C = np.asarray(counts, dtype=np.int64)
    remap = np.zeros(256, dtype=np.int64)
    for pred_i, target_i in match:
        if int(pred_i) < 256:
            remap[int(pred_i)] = int(target_i)
    rows = C.sum(1)
    jac = []
    for i in range(n_classes):
        sel = remap == i
        tp = int(C[sel, i].sum())
        fp = int(rows[sel].sum()) - tp
        fn = int(C[:, i].sum()) - tp
        jac.append(float(tp) / max(float(tp + fp + fn), 1e-8))
    return {"jaccards_all_categs": jac, "mIoU": np.mean(jac)}


def object_metrics(counts) -> Tuple[list, list]:
    """compute_accuracy / compute_iou (metrics.py:65-76) of every image from its {TP, FP, FN, TN}: acc = fp32
    count / numel, IoU = fp32 tp / union with 0 / 0 -> 0 (an int, as the reference's NaN test gives). Exact while an
    image has fewer than 2^24 pixels (the reference's fp32 sum is exact there)."""
    acc, iou = [], []
    for tp, fp, fn, tn in np.asarray(counts, dtype=np.int64).tolist():
        acc.append(float(np.float32(tp + tn) / np.float32(tp + fp + fn + tn)))
        union = tp + fp + fn
        iou.append(float(np.float32(tp) / np.float32(union)) if union else 0)
    return acc, iou


def mean(x):
    """metrics.mean: Python's sequential sum over the per-image values."""
    return sum(x) / len(x)


# ------------------------------------------------------------------------------------------------ overrides
def _value(s: str):
    if s in ("null", "None", "~"):
        return None
    if s in ("true", "True"):
        return True
    if s in ("false", "False"):
        return False
    if len(s) >= 2 and s[0] == s[-1] and s[0] in "'\"":
        return s[1:-1]
    try:
        return int(s)
    except ValueError:
        return s


def parse_overrides(argv: Sequence[str], defaults: Dict[str, object], extra=lambda key: False) -> Dict[str, object]:
    """Hydra-style ``key=value`` overrides (``+key=value`` too) of the keys in defaults (or accepted by extra);
    anything else is a ValueError."""
    cfg = dict(defaults)
    for a in argv:
        if "=" not in a:
            raise ValueError(f"{a!r}: overrides are key=value")
        key, val = a.split("=", 1)
        key = key.lstrip("+")
        if key not in defaults and not extra(key):
            raise ValueError(f"unknown override {key!r}: known keys are {', '.join(sorted(defaults))}")
        cfg[key] = _value(val)
    if cfg.get("wandb"):
        raise ValueError("wandb=True is not supported (no Weights & Biases logging here)")
    if cfg.get("cpu"):
        raise ValueError("cpu=True is not supported: the counts run on the GPU only")
    return cfg


def _common_defaults():
    return {"name": "debug", "seed": 1, "fp16": False, "cpu": False, "wandb": False}


def _map_threads(fn, items):
    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        return list(ex.map(fn, items))


def _read_u8(path, convert: Optional[str] = None) -> np.ndarray:
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im.convert(convert) if convert else im)


def _header(path) -> Tuple[Tuple[int, int], str]:
    """((H, W), mode) from the file header, without decoding the pixels."""
    from PIL import Image
    with Image.open(path) as im:
        return (im.size[1], im.size[0]), im.mode


# ------------------------------------------------------------------------------------------------ semantic command
def semantic_defaults() -> Dict[str, object]:
    """config/base.yaml + config/eval.yaml, the keys evaluate() reads."""
    return {**_common_defaults(), "job_type": "eval",
            "segments_dir": "", "data.num_classes": 20,
            "data.val_kwargs.root": os.path.expanduser("~") + "/machine-learning-datasets/semantic-segmentation/"
                                                             "PASCAL_VOC/VOC2012",
            "data.val_kwargs.year": "2012", "data.val_kwargs.image_set": "val", "data.val_kwargs.download": False,
            "n_clusters": None}


def voc_pairs(root: str, year: str, image_set: str, segments_dir: str):
    """VOCSegmentationWithPseudolabels (dataset/voc.py:22-131) for a split file: (images, targets, segments) and the
    reference's "Loaded segments" lines. Segment files are paired by position with all JPEGImages, both sorted, then
    filtered to the split."""
    from torchvision.datasets.voc import DATASET_YEAR_DICT
    year, image_set = str(year), str(image_set)
    if year == "2007-test":
        if image_set != "test":
            raise ValueError("In the test image set of the year 2007 only image_set='test' is allowed. "
                             "For all other image sets use year='2007' instead.")
        year = "2007"
    valid = ["trainval", "val"] + (["test"] if year == "2007" else [])
    if image_set == "train":
        raise ValueError("data.val_kwargs.image_set=train is not supported: the reference pairs every train image "
                         "with one arbitrary target")
    if image_set not in valid:
        raise ValueError(f"Unknown value '{image_set}' for argument image_set. Valid values are {{{', '.join(valid)}}}.")
    if year not in DATASET_YEAR_DICT:
        raise ValueError(f"data.val_kwargs.year={year}: unknown VOC year")
    key = "2007-test" if year == "2007" and image_set == "test" else year
    root = os.path.expanduser(root)
    voc_root = os.path.join(root, DATASET_YEAR_DICT[key]["base_dir"])
    if not os.path.isdir(voc_root):
        raise RuntimeError("Dataset not found or corrupted. You can use download=True to download it")
    split_f = os.path.join(voc_root, "ImageSets", "Segmentation", image_set.rstrip("\n") + ".txt")
    with open(split_f) as f:
        file_names = [x.strip() for x in f.readlines()]
    image_dir = os.path.join(voc_root, "JPEGImages")
    images = [os.path.join(image_dir, x + ".jpg") for x in file_names]
    targets = [os.path.join(voc_root, "SegmentationClass", x + ".png") for x in file_names]
    all_segment_files = sorted(map(str, Path(segments_dir).iterdir()))
    all_img_files = sorted(Path(images[0]).parent.iterdir())
    assert len(all_img_files) == len(all_segment_files), (len(all_img_files), len(all_segment_files))
    valid_img_stems = set([Path(p).stem for p in images])
    segments = [all_segment_files[i] for i, p in enumerate(all_img_files) if p.stem in valid_img_stems]
    assert len(segments) == len(images), f'{len(segments)=} and {len(images)=}'
    lines = ["Loaded segments and images", f"First image filepath: {images[0]}",
             f"First segmap filepath: {segments[0]}", f"Last image filepath: {images[-1]}",
             f"Last segmap filepath: {segments[-1]}"]
    return images, targets, segments, lines


def _label_header(path) -> Tuple[int, int]:
    shape, mode = _header(path)
    if mode not in ("L", "P"):
        raise ValueError(f"{path}: PNG mode {mode} is not a uint8 label map (L or P)")
    return shape


def semantic_main(argv=None, out=None) -> Tuple[dict, object]:
    """semantic-segmentation/eval.py: prints the reference's lines and returns (eval_stats, match)."""
    out = out or sys.stdout
    cfg = parse_overrides(list(argv or []), semantic_defaults())
    if cfg["data.val_kwargs.download"]:
        raise ValueError("data.val_kwargs.download=True is not supported (no network access here)")
    n_classes = int(cfg["data.num_classes"]) + 1
    n_clusters = n_classes if cfg["n_clusters"] is None else int(cfg["n_clusters"])
    if not 1 <= n_classes <= MAX_CLASSES:
        raise ValueError(f"data.num_classes={cfg['data.num_classes']}: up to {MAX_CLASSES - 1} classes are supported")
    if n_clusters < 1:
        raise ValueError(f"n_clusters={n_clusters} must be >= 1")
    images, targets, segments, lines = voc_pairs(cfg["data.val_kwargs.root"], cfg["data.val_kwargs.year"],
                                                 cfg["data.val_kwargs.image_set"], str(cfg["segments_dir"]))
    for line in lines:
        print(line, file=out)

    # headers only, before any device work: every shape mismatch is reported here
    def plan(i):
        return semantic_gather(_label_header(segments[i]), _header(images[i])[0], _label_header(targets[i]),
                               segments[i])
    gathers = _map_threads(plan, range(len(images)))

    counts = semantic_counts([], n_classes)
    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        for s in range(0, len(images), BATCH):
            idx = range(s, min(s + BATCH, len(images)))
            maps = list(ex.map(lambda i: (_read_u8(segments[i]), _read_u8(targets[i])), idx))
            semantic_counts([(p, t, gathers[i]) for (p, t), i in zip(maps, idx)], n_classes, counts)
    C = counts.cpu().numpy()

    print("Using hungarian algorithm for matching" if n_clusters == n_classes else
          "Using majority voting for matching", file=out)
    if n_clusters == n_classes:
        print("Using iou as metric", file=out)
    match = match_clusters(C, n_clusters, n_classes)
    print(f"Optimal matching: {match}", file=out)
    eval_stats = semantic_miou(C, match, n_classes)
    print("Evaluation of semantic segmentation ", file=out)
    print("mIoU is %.2f" % (100 * eval_stats["mIoU"]), file=out)
    print(eval_stats, file=out)
    return eval_stats, match


# ------------------------------------------------------------------------------------------------ object command
OBJECT_DATASETS = {   # config/eval.yaml: name -> (images_dir, labels_dir, crop, prediction sub-directory)
    "CUB": ("CUB_200_2011/test_images", "CUB_200_2011/test_segmentations", True, "CUB_200_2011"),
    "DUT_OMRON": ("DUT_OMRON/DUT-OMRON-image", "DUT_OMRON/pixelwiseGT-new-PNG", False, "DUT_OMRON"),
    "DUTS": ("DUTS/DUTS-TE/DUTS-TE-Image", "DUTS/DUTS-TE/DUTS-TE-Mask", False, "DUTS"),
    "ECSSD": ("ECSSD/images", "ECSSD/ground_truth_mask", False, "ECSSD"),
}
IMG_EXTENSIONS = ('.jpg', '.jpeg', '.png', '.ppm', '.bmp', '.pgm', '.tif', '.tiff', '.webp')
PRED_VALUE_SETS = [{0, 255}, {0, 1}, {0}]


def object_defaults() -> Dict[str, object]:
    return {**_common_defaults(), "job_type": "eval", "data_root": os.environ.get("GANSEG_DATA_SEG_ROOT"),
            "predictions.root": "/path/to/object-segmentation-data", "predictions.run": "run_name",
            "predictions.downsample": 16, "datasets": ",".join(OBJECT_DATASETS)}


def object_files(images_dir: str, labels_dir: str) -> Tuple[List[Path], List[Path]]:
    """SegmentationDataset (dataset.py:27-54): the class-folder vs flat test on the first directory entry, then
    sorted images and labels paired by position."""
    has_folders = not any(str(next(Path(images_dir).iterdir())).endswith(ext) for ext in IMG_EXTENSIONS)
    if has_folders:
        image_paths = [p for f in Path(images_dir).iterdir() for p in f.iterdir()]
        label_paths = [p for f in Path(labels_dir).iterdir() for p in f.iterdir()]
    else:
        image_paths, label_paths = Path(images_dir).iterdir(), Path(labels_dir).iterdir()
    image_paths, label_paths = list(sorted(image_paths)), list(sorted(label_paths))
    assert len(image_paths) == len(label_paths)
    return image_paths, label_paths


def read_prediction(path) -> np.ndarray:
    """main.py:84-86: the file as mode L, values {0, 255}, {0, 1} or {0} (else a ValueError naming the file), 255 -> 1."""
    preds = np.array(_read_u8(path, "L"))
    values = set(np.unique(preds).tolist())
    if values not in PRED_VALUE_SETS:
        raise ValueError(f"{path}: prediction values {sorted(values)} are not one of {{0, 255}}, {{0, 1}} or {{0}}")
    preds[preds == 255] = 1
    return preds


def read_mask_plane(path) -> np.ndarray:
    """The R channel of mask.convert('RGB') (dataset.py:83): ToTensor() > 0.5 is R >= 128."""
    return np.ascontiguousarray(_read_u8(path, "RGB")[..., 0])


def object_main(argv=None, out=None) -> Dict[str, Dict[str, float]]:
    """object-segmentation/main.py: prints ``[{name}] acc: {value}`` and ``[{name}] iou: {value}`` for every selected
    data set and returns {name: {'acc': value, 'iou': value}}."""
    out = out or sys.stdout
    cfg = parse_overrides(list(argv or []), object_defaults(),
                          extra=lambda k: k.startswith("predictions.") and k.split(".", 1)[1] in OBJECT_DATASETS)
    if cfg["job_type"] != "eval":
        raise ValueError(f"job_type={cfg['job_type']}: only eval is implemented (the reference raises too)")
    names = [n for n in str(cfg["datasets"]).split(",") if n]
    for n in names:
        if n not in OBJECT_DATASETS:
            raise ValueError(f"datasets={cfg['datasets']}: {n!r} is not one of {', '.join(OBJECT_DATASETS)}")
    ds = cfg["predictions.downsample"]
    if ds is not None and (not isinstance(ds, int) or isinstance(ds, bool) or ds < 1):
        raise ValueError(f"predictions.downsample={ds}: a positive integer or null")
    if cfg["data_root"] is None:
        raise ValueError("data_root: set GANSEG_DATA_SEG_ROOT or pass data_root=<dir>")

    # every data set is checked before any device work: file pairing, prediction value sets, shapes
    plans = []
    for name in names:
        img_sub, lab_sub, crop, pred_sub = OBJECT_DATASETS[name]
        pred_dir = cfg.get(f"predictions.{name}") or f"{cfg['predictions.root']}/{pred_sub}/{cfg['predictions.run']}"
        image_paths, label_paths = object_files(f"{cfg['data_root']}/{img_sub}", f"{cfg['data_root']}/{lab_sub}")
        pred_files = [os.path.join(str(pred_dir), f"{p.stem}.png") for p in image_paths]

        def plan(j, pred_files=pred_files, label_paths=label_paths, crop=crop):
            shape = read_prediction(pred_files[j]).shape
            return object_gather(shape, _header(label_paths[j])[0], ds, crop, pred_files[j])
        plans.append((name, pred_files, label_paths, _map_threads(plan, range(len(pred_files)))))

    results = {}
    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        for name, pred_files, label_paths, gathers in plans:
            acc, iou = [], []
            for s in range(0, len(pred_files), BATCH):
                idx = range(s, min(s + BATCH, len(pred_files)))
                maps = list(ex.map(lambda j: (read_prediction(pred_files[j]), read_mask_plane(label_paths[j])), idx))
                a, u = object_metrics(object_counts([(p, t, gathers[j]) for (p, t), j in zip(maps, idx)]))
                acc += a
                iou += u
            results[name] = {"acc": mean(acc), "iou": mean(iou)}
            for metric_name, value in results[name].items():
                print(f"[{name}] {metric_name}: {value}", file=out)
    return results
