"""Object localization (the reference's object-localization/main.py with object_discovery.py and datasets.py): boxes
from the eigenvectors (eigen-segmentation), and the LOST and DINO-seg baselines, scored by CorLoc on Pascal VOC and
COCO20k.

Device work: csrc/localize.cu (the three box kernels, one CTA per image) and the last-block ViT outputs of csrc/vit.cu
(zero-padded grid, q / k / v features, the CLS attention row). LOST and DINO-seg run ``--batch_size`` images per ViT
forward in list order whatever their sizes (a ragged forward with outputs padded to the batch's largest grid, then one
box kernel over the batch); eigen-segmentation from images batches images of one size. The host reads VOC annotations
with ElementTree and the COCO20k selection with json, JPEG sizes from their headers and images on reader threads, and
keeps the reference's output files: ``{output_dir}/{dataset}/{exp_name}/preds.pkl``, ``gt.pkl`` (dict image name ->
int64 boxes [xmin, ymin, xmax, ymax]; the VOC file name or the COCO image id) and ``results.txt``. Single process:
there is no multi-GPU sharding of this command."""
from __future__ import annotations

import argparse
import json
import os
import pickle
import sys
import xml.etree.ElementTree as ET
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from pprint import pprint
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, io_pipeline, spectral
from . import vit as vit_mod

SEGMENT_INDEX = {"matting": 1, "laplacian": 1, "affinity": 0}   # main.py:270
DINOSEG_THRESHOLD = 0.6                                         # object_discovery.py:236 (official_th)


# ------------------------------------------------------------------------------------------------ box kernels
@torch.no_grad()
def eigseg_boxes(evecs: torch.Tensor, which: int, sizes: Sequence[Tuple[int, int]]):
    """get_bbox_from_patch_mask for a batch: row ``which`` of evecs [B, K, N] fp32 CUDA; sizes = the un-cropped
    (H, W) of every image. Returns (boxes int64 [B, 4], status int32 [B]) as numpy."""
    _lib.require_cuda(evecs, "evecs")
    ev = evecs.to(torch.float32).contiguous()
    B, K, N = ev.shape
    assert len(sizes) == B
    lib = _lib.load()
    dims = torch.tensor([[int(h), int(w)] for h, w in sizes], dtype=torch.int32).contiguous()
    with torch.cuda.device(ev.device):
        boxes = torch.empty(B, 4, dtype=torch.int32, device=ev.device)
        status = torch.empty(B, dtype=torch.int32, device=ev.device)
        ws = spectral._scratch.get("eigseg", int(lib.dss_eigseg_boxes_workspace_bytes(B)), ev.device)
        _lib.check(lib.dss_eigseg_boxes(ev.data_ptr(), B, K, N, int(which), dims.data_ptr(), boxes.data_ptr(),
                                        status.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(ev.device)),
                   "dss_eigseg_boxes")
    return boxes.cpu().numpy().astype(np.int64), status.cpu().numpy()


@torch.no_grad()
def lost_boxes(feats: torch.Tensor, grid: Tuple[int, int], size: Tuple[int, int], patch: int, k_patches: int = 100):
    """LOST for a batch of images of one size: feats [B, N, d] fp32 CUDA on the grid (gh, gw) (the zero-padded one in
    the reference), size = the un-padded (H, W). A = F F^T comes from the affinity kernel without any normalisation.
    Returns (boxes int64 [B, 4], seeds int32 [B], status int32 [B]) as numpy."""
    _lib.require_cuda(feats, "feats")
    B, N, _ = feats.shape
    A = spectral.affinity(feats, normalize=False, threshold_at_zero=False, scale_by_max=False)
    lib = _lib.load()
    with torch.cuda.device(A.device):
        boxes = torch.empty(B, 4, dtype=torch.int32, device=A.device)
        seeds = torch.empty(B, dtype=torch.int32, device=A.device)
        status = torch.empty(B, dtype=torch.int32, device=A.device)
        ws = spectral._scratch.get("lost", int(lib.dss_lost_workspace_bytes(B, N)), A.device)
        _lib.check(lib.dss_lost_boxes(A.data_ptr(), B, N, A.shape[2], int(grid[0]), int(grid[1]), int(size[0]),
                                      int(size[1]), int(patch), int(k_patches), boxes.data_ptr(), seeds.data_ptr(),
                                      status.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(A.device)),
                   "dss_lost_boxes")
    return boxes.cpu().numpy().astype(np.int64), seeds.cpu().numpy(), status.cpu().numpy()


@torch.no_grad()
def dinoseg_boxes(cls_attn: torch.Tensor, grid: Tuple[int, int], patch: int, head: int = 4):
    """dino_seg for a batch: cls_attn [B, heads, N] fp32 CUDA on the grid (gh, gw). Returns (boxes int64 [B, 4],
    status int32 [B]) as numpy."""
    _lib.require_cuda(cls_attn, "cls_attn")
    a = cls_attn.to(torch.float32).contiguous()
    B, heads, N = a.shape
    with torch.cuda.device(a.device):
        boxes = torch.empty(B, 4, dtype=torch.int32, device=a.device)
        status = torch.empty(B, dtype=torch.int32, device=a.device)
        _lib.check(_lib.load().dss_dinoseg_boxes(a.data_ptr(), B, heads, N, int(head), int(grid[0]), int(grid[1]),
                                                 int(patch), boxes.data_ptr(), status.data_ptr(),
                                                 _lib.stream_ptr(a.device)), "dss_dinoseg_boxes")
    return boxes.cpu().numpy().astype(np.int64), status.cpu().numpy()


@torch.no_grad()
def lost_boxes_ragged(feats: torch.Tensor, grids: Sequence[Tuple[int, int]], sizes: Sequence[Tuple[int, int]],
                      patch: int, k_patches: int = 100):
    """LOST for a batch of images of any sizes: feats [B, n_max, d] fp32 CUDA in the padded layout of
    DinoViT.forward_last_ragged (image b's gh_b * gw_b rows first, then zero rows), grids[b] = (gh_b, gw_b), sizes[b] =
    the un-padded (H_b, W_b). One affinity over the padded batch: the zero rows leave each image's block as the image
    alone gives it. Returns (boxes int64 [B, 4], seeds int32 [B], status int32 [B]) as numpy, each image's as
    lost_boxes gives for that image alone."""
    _lib.require_cuda(feats, "feats")
    B, n_max, _ = feats.shape
    assert len(grids) == B and len(sizes) == B
    A = spectral.affinity(feats, normalize=False, threshold_at_zero=False, scale_by_max=False)
    lib = _lib.load()
    dims = torch.tensor([[int(g[0]), int(g[1]), int(s[0]), int(s[1])] for g, s in zip(grids, sizes)], dtype=torch.int32)
    with torch.cuda.device(A.device):
        boxes = torch.empty(B, 4, dtype=torch.int32, device=A.device)
        seeds = torch.empty(B, dtype=torch.int32, device=A.device)
        status = torch.empty(B, dtype=torch.int32, device=A.device)
        ws = spectral._scratch.get("lost", int(lib.dss_lost_ragged_workspace_bytes(B, n_max)), A.device)
        _lib.check(lib.dss_lost_boxes_ragged(A.data_ptr(), B, n_max, A.shape[2], dims.data_ptr(), int(patch),
                                             int(k_patches), boxes.data_ptr(), seeds.data_ptr(), status.data_ptr(),
                                             ws.data_ptr(), ws.numel(), _lib.stream_ptr(A.device)),
                   "dss_lost_boxes_ragged")
    return boxes.cpu().numpy().astype(np.int64), seeds.cpu().numpy(), status.cpu().numpy()


@torch.no_grad()
def dinoseg_boxes_ragged(cls_attn: torch.Tensor, grids: Sequence[Tuple[int, int]], patch: int, head: int = 4):
    """dino_seg for a batch of images of any sizes: cls_attn [B, heads, n_max] fp32 CUDA in the padded layout of
    DinoViT.forward_last_ragged, grids[b] = (gh_b, gw_b). Returns (boxes int64 [B, 4], status int32 [B]) as numpy."""
    _lib.require_cuda(cls_attn, "cls_attn")
    a = cls_attn.to(torch.float32).contiguous()
    B, heads, n_max = a.shape
    assert len(grids) == B
    lib = _lib.load()
    dims = torch.tensor([[int(g[0]), int(g[1])] for g in grids], dtype=torch.int32)
    with torch.cuda.device(a.device):
        boxes = torch.empty(B, 4, dtype=torch.int32, device=a.device)
        status = torch.empty(B, dtype=torch.int32, device=a.device)
        ws = spectral._scratch.get("dinoseg", int(lib.dss_dinoseg_ragged_workspace_bytes(B)), a.device)
        _lib.check(lib.dss_dinoseg_boxes_ragged(a.data_ptr(), B, heads, n_max, int(head), dims.data_ptr(), int(patch),
                                                boxes.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(),
                                                _lib.stream_ptr(a.device)), "dss_dinoseg_boxes_ragged")
    return boxes.cpu().numpy().astype(np.int64), status.cpu().numpy()


def raise_for_status(status: int, name: str, N: int = 0, size=None) -> None:
    """The reference's exceptions for a failed image."""
    if status == _lib.LOC_NO_GRID:
        raise ValueError(f"{name}: no patch grid of the image size {size} has {N} cells")
    if status == _lib.LOC_SEED_IN_BACKGROUND:
        raise ValueError("The seed is in the background component.")
    if status == _lib.LOC_EMPTY_COMPONENT:
        raise ValueError(f"{name}: DINO-seg selected an empty component (every patch is kept)")
    if status != _lib.LOC_OK:
        raise RuntimeError(f"{name}: unknown localization status {status}")


# ------------------------------------------------------------------------------------------------ VOC and CorLoc
VOC_YEARS = {"VOC07": "2007", "VOC12": "2012"}


def voc_root(dataset_root: str, year: str) -> Path:
    """torchvision's VOCDetection layout under the reference's data-set directory: {root}/VOCdevkit/VOC{year}."""
    return Path(dataset_root) / "VOCdevkit" / f"VOC{year}"


def read_voc_list(root: Path, image_set: str) -> List[str]:
    with open(root / "ImageSets" / "Main" / f"{image_set}.txt") as f:
        return [x.strip() for x in f.readlines()]


def parse_voc_xml(path) -> dict:
    """The fields of VOCDetection's target that the localization reads: {'filename', 'size': {'width', 'height'},
    'object': [{'name', 'truncated', 'difficult', 'bndbox': {'xmin', 'ymin', 'xmax', 'ymax'}}]}, values as strings."""
    ann = ET.parse(path).getroot()
    out = {"filename": (ann.findtext("filename") or "").strip(), "object": []}
    size = ann.find("size")
    if size is not None:
        out["size"] = {k: (size.findtext(k) or "").strip() for k in ("width", "height", "depth")}
    for o in ann.findall("object"):
        obj = {k: (o.findtext(k) or "").strip() for k in ("name", "truncated", "difficult")}
        bb = o.find("bndbox")
        obj["bndbox"] = {k: (bb.findtext(k) or "").strip() for k in ("xmin", "ymin", "xmax", "ymax")}
        out["object"].append(obj)
    return out


def extract_gt_voc(ann: dict, remove_hards: bool = False):
    """datasets.py:238-266: boxes int64 [n, 4] with xmin / ymin shifted by -1 (1-based inclusive pixel indices to
    0-based edges); remove_hards drops truncated or difficult objects."""
    boxes, classes = [], []
    for o in ann["object"]:
        if remove_hards and (o.get("truncated") == "1" or o.get("difficult") == "1"):
            continue
        classes.append(o["name"])
        b = o["bndbox"]
        boxes.append([int(b["xmin"]) - 1, int(b["ymin"]) - 1, int(b["xmax"]), int(b["ymax"])])
    return np.asarray(boxes), classes


def extract_gt_coco(anns: Sequence[dict]) -> np.ndarray:
    """datasets.py:218-235: int64 boxes [n, 4] of the non-crowd annotations in their JSON order; COCO's float
    [x, y, w, h] becomes [x, y, x + w, y + h], each rounded half to even by Python's round on float64."""
    boxes = []
    for a in anns:
        if a["iscrowd"] == 1:
            continue
        x, y, w, h = (float(v) for v in a["bbox"])
        boxes.append([int(round(v)) for v in (x, y, x + w, y + h)])
    return np.asarray(boxes, dtype=np.int64).reshape(-1, 4)


# COCO20k: the reference's layout under the data-set directory (datasets.py:50-66)
COCO_IMAGES = Path("COCO") / "images" / "train2014"
COCO_ALL_ANNOTATIONS = Path("COCO") / "annotations" / "instances_train2014.json"
COCO_SELECTION_LIST = "coco_20k_filenames.txt"
COCO_SELECTION_CACHE = "instances_train2014_sel20k.json"


def read_coco20k_ids(path) -> List[int]:
    """The image ids of the selection list in list order, each once: ``COCO_train2014_000000000123.jpg`` -> 123."""
    with open(path) as f:
        ids = [int(line.replace("\n", "").split("_")[-1].split(".")[0]) for line in f if line.strip()]
    return list(dict.fromkeys(ids))


def _check_coco20k_cache(sel: dict, ids: Sequence[int], path) -> None:
    fix = f"{path}: delete it so that it is rebuilt from the full train2014 annotations"
    images, anns = sel.get("images"), sel.get("annotations")
    if (not isinstance(images, list) or not isinstance(anns, list) or "categories" not in sel
            or any(not isinstance(im, dict) or "file_name" not in im for im in images)
            or any(not isinstance(a, dict) for a in anns)):
        raise ValueError(f"{fix}: it is not a COCO annotation file of image records (the format the reference's "
                         "select_coco_20k writes holds annotations where image records belong)")
    if sorted(im["id"] for im in images) != sorted(ids):
        raise ValueError(f"{fix}: its image ids differ from the selection list's")


def select_coco20k(root) -> dict:
    """The COCO20k annotations: the cache ``{root}/instances_train2014_sel20k.json`` if it exists (checked against the
    selection list, never overwritten), else built from the full train2014 file and written there. The cache is a COCO
    file: the selected image records in list order, every annotation of those images in the full file's order, and
    the full file's categories."""
    root = Path(root)
    ids = read_coco20k_ids(root / COCO_SELECTION_LIST)
    cache = root / COCO_SELECTION_CACHE
    if cache.exists():
        with open(cache) as f:
            sel = json.load(f)
        _check_coco20k_cache(sel, ids, cache)
        return sel
    with open(root / COCO_ALL_ANNOTATIONS) as f:
        full = json.load(f)
    records = {im["id"]: im for im in full["images"]}
    missing = [i for i in ids if i not in records]
    if missing:
        raise ValueError(f"{root / COCO_SELECTION_LIST}: image id {missing[0]} has no image record in "
                         f"{root / COCO_ALL_ANNOTATIONS}")
    wanted = set(ids)
    sel = {"images": [records[i] for i in ids], "annotations": [a for a in full["annotations"] if a["image_id"] in wanted],
           "categories": full["categories"]}
    text = json.dumps(sel)
    with open(cache, "x") as f:   # "x": a cache another process wrote meanwhile is not overwritten
        f.write(text)
    return sel


def coco20k_targets(sel: dict) -> List[Tuple[dict, List[dict]]]:
    """(image record, annotations) per image in torchvision's CocoDetection order: ascending image id, each image's
    annotations in file order (pycocotools' getAnnIds / loadAnns)."""
    anns: Dict[int, List[dict]] = {}
    for a in sel["annotations"]:
        anns.setdefault(a["image_id"], []).append(a)
    return [(im, anns.get(im["id"], [])) for im in sorted(sel["images"], key=lambda im: im["id"])]


def bbox_iou(box1: torch.Tensor, box2: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    """IoU of box1 [4] with each row of box2 [n, 4] in the reference's arithmetic (datasets.py:269-294): torch ops on
    the int64 boxes, eps added to each height and to the union, so the result is float32 exactly as the reference's.
    A CorLoc decision at IoU 0.5 therefore agrees with it to the last bit."""
    b2 = box2.T
    inter = ((torch.min(box1[2], b2[2]) - torch.max(box1[0], b2[0])).clamp(0)
             * (torch.min(box1[3], b2[3]) - torch.max(box1[1], b2[1])).clamp(0))
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1] + eps
    w2, h2 = b2[2] - b2[0], b2[3] - b2[1] + eps
    union = w1 * h1 + w2 * h2 - inter + eps
    return inter / union


def corloc_hit(pred: np.ndarray, gt: np.ndarray) -> bool:
    return bool(torch.any(bbox_iou(torch.from_numpy(np.asarray(pred)), torch.from_numpy(np.asarray(gt))) >= 0.5))


def jpeg_size(path) -> Tuple[int, int]:
    """(H, W) from the image header, without decoding the pixels."""
    from PIL import Image
    with Image.open(path) as im:
        W, H = im.size
    return H, W


def load_rgb(path) -> np.ndarray:
    """uint8 [H, W, 3]: PIL ``.convert("RGB")``, as the reference's loader decodes."""
    from PIL import Image
    with open(path, "rb") as f:
        return np.asarray(Image.open(f).convert("RGB"))


# ------------------------------------------------------------------------------------------------ command line
ARCH_MAP = {("vit_small", 16): "dino_vits16", ("vit_small", 8): "dino_vits8", ("vit_base", 16): "dino_vitb16",
            ("vit_base", 8): "dino_vitb8"}


def parse_args(argv=None):
    """The reference's parse_args (main.py:26-131), plus --dataset_root, --checkpoint, --random_init / --seed and
    --batch_size."""
    parser = argparse.ArgumentParser("Visualize Self-Attention maps")
    parser.add_argument("--arch", default="vit_small", type=str,
                        choices=["vit_tiny", "vit_small", "vit_base", "resnet50", "vgg16_imagenet", "resnet50_imagenet"],
                        help="Model architecture (vit_small and vit_base are supported).")
    parser.add_argument("--patch_size", default=16, type=int, help="Patch resolution of the model.")
    parser.add_argument("--dataset", default="VOC07", type=str, choices=[None, "VOC07", "VOC12", "COCO20k"],
                        help="Dataset name.")
    parser.add_argument("--set", default="trainval", type=str, choices=["val", "train", "trainval", "test"],
                        help="Path of the image to load.")
    parser.add_argument("--image_path", type=str, default=None,
                        help="If want to apply only on one image, give file path.")
    parser.add_argument("--output_dir", type=str, default="outputs",
                        help="Output directory to store predictions and visualizations.")
    parser.add_argument("--no_hard", action="store_true", help="Only used in the case of the VOC_all setup (see the paper).")
    parser.add_argument("--no_evaluation", action="store_true", help="Compute the evaluation.")
    parser.add_argument("--save_predictions", default=True, type=bool, help="Save predicted bouding boxes.")
    parser.add_argument("--visualize", type=str, choices=["fms", "seed_expansion", "pred", None], default=None,
                        help="Not supported here.")
    parser.add_argument("--resnet_dilate", type=int, default=2, help="Dilation level of the resnet model.")
    parser.add_argument("--which_features", type=str, default="k", choices=["k", "q", "v"], help="Which features to use")
    parser.add_argument("--k_patches", type=int, default=100,
                        help="Number of patches with the lowest degree considered.")
    parser.add_argument("--name", type=str, default=None, help="Experiment name")
    parser.add_argument("--skip_if_exists", action="store_true", help="If results dir already exists , exit")
    parser.add_argument("--dinoseg", action="store_true", help="Apply DINO-seg baseline.")
    parser.add_argument("--dinoseg_head", type=int, default=4)
    parser.add_argument("--eigenseg", action="store_true", help="Apply eigenvalue method")
    parser.add_argument("--precomputed_eigs_dir", default=None, type=str,
                        help="Apply eigenvalue method with precomputed bboxes")
    parser.add_argument("--precomputed_eigs_downsample", default=16, type=str)
    parser.add_argument("--which_matrix", choices=["infer", "affinity", "laplacian"], default="infer",
                        help="Which matrix to use for eigenvector calculation")
    # additions of this implementation
    parser.add_argument("--dataset_root", type=str, default=None,
                        help="Data-set directory, by default the one the reference hard-codes in the working "
                             "directory. VOC07 / VOC12: datasets/VOC2007 or datasets/VOC2012, holding "
                             "VOCdevkit/VOC<year>/. COCO20k: datasets, holding COCO/images/train2014/, "
                             "COCO/annotations/instances_train2014.json, coco_20k_filenames.txt and the selection "
                             "cache instances_train2014_sel20k.json (written on the first run).")
    parser.add_argument("--checkpoint", type=str, default=None,
                        help="DINO weights (.pth). Default: $DSS_DINO_CHECKPOINT or the torch.hub cache. Note: for "
                             "vit_small/8 the reference loads dino_deitsmall8_300ep_pretrain.pth, not the hub file "
                             "dino_deitsmall8_pretrain.pth: pass it here to reproduce its numbers.")
    parser.add_argument("--random_init", action="store_true", help="Use randomly initialised weights (tests only).")
    parser.add_argument("--seed", type=int, default=None, help="Seed of the random weights (implies --random_init).")
    parser.add_argument("--batch_size", type=int, default=16,
                        help="Images per ViT batch: LOST and DINO-seg take them in list order whatever their sizes; "
                             "--eigenseg from images batches images of one size.")
    parser.add_argument("--precision", type=str, default="fp16", choices=["fp16", "fp32"],
                        help="ViT arithmetic: fp16 operands (fast) or split-fp16 operands with the fp32 model's results.")
    args = parser.parse_args(argv)
    if args.image_path is not None:
        args.save_predictions = False
        args.no_evaluation = True
        args.dataset = None
    return args


def check_supported(args) -> None:
    """Reject what this implementation does not run, before any work."""
    if args.arch in ("resnet50", "vgg16_imagenet", "resnet50_imagenet"):
        raise ValueError(f"--arch {args.arch}: the CNN backbones have no kernels here (only vit_small / vit_base)")
    if args.arch == "vit_tiny":
        raise ValueError("--arch vit_tiny: embedding dim 192 is not a supported ViT (384 or 768)")
    if (args.arch, args.patch_size) not in ARCH_MAP:
        raise ValueError(f"--arch {args.arch} --patch_size {args.patch_size}: patch size must be 8 or 16")
    if args.visualize:
        raise ValueError("--visualize is not supported (it needs skimage and writes matplotlib figures)")
    if args.dataset == "COCO20k" and args.set != "train":
        raise ValueError(f"--dataset COCO20k --set {args.set}: COCO20k is a selection of train2014, pass --set train")
    if args.dinoseg and args.eigenseg:
        raise ValueError("--dinoseg and --eigenseg are exclusive (the reference runs DINO-seg and ignores --eigenseg)")
    if args.eigenseg and args.precomputed_eigs_dir is None and args.which_matrix == "infer":
        raise ValueError("--which_matrix infer needs --precomputed_eigs_dir (it reads the matrix from the directory "
                         "name); pass affinity or laplacian")
    if args.k_patches < 1:
        raise ValueError("--k_patches must be >= 1")


def experiment_name(args) -> str:
    if args.name is not None:
        return args.name
    if args.dinoseg:
        return f"{args.arch}-{args.patch_size}_dinoseg-head{args.dinoseg_head}"
    return f"LOST-{args.arch}{args.patch_size}_{args.which_features}"


class _Item:
    __slots__ = ("name", "path", "gt", "eig_file")

    def __init__(self, name, path, gt, eig_file=None):
        self.name, self.path, self.gt = name, path, gt
        self.eig_file = eig_file if eig_file is not None else name.replace(".jpg", ".pth")   # main.py:255-258


def _dataset_items(args):
    """(data-set name, [items]) in list order; images whose GT is empty under --no_hard are dropped (main.py:245-249)."""
    if args.image_path is not None:
        return args.image_path.split("/")[-1], [_Item(args.image_path.split("/")[-1].split(".")[0], args.image_path, None)]
    if args.dataset == "COCO20k":
        return _coco20k_items(args)
    year = VOC_YEARS[args.dataset]
    root_dir = args.dataset_root or f"datasets/VOC{year}"
    if not os.path.exists(root_dir):
        raise ValueError(f"{root_dir}: please follow the README to set up the datasets (or pass --dataset_root)")
    root = voc_root(root_dir, year)
    ids = read_voc_list(root, args.set)
    name = f"{args.dataset}_{args.set}" + ("-nohards" if args.no_hard else "")
    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        anns = list(ex.map(lambda i: parse_voc_xml(root / "Annotations" / f"{i}.xml"), ids))
    items = []
    for i, ann in zip(ids, anns):
        gt = None
        if not args.no_evaluation:
            gt, _ = extract_gt_voc(ann, remove_hards=args.no_hard)
            if gt.shape[0] == 0 and args.no_hard:
                continue
        items.append(_Item(ann["filename"], str(root / "JPEGImages" / f"{i}.jpg"), gt))
    return name, items


def _coco20k_items(args):
    """COCO20k in CocoDetection order, named by image id. An image without a non-crowd box is dropped under --no_hard
    (as the reference drops it); without --no_hard it is refused here, before any device work, where the reference
    crashes in bbox_iou or get_image_name."""
    root_dir = args.dataset_root or "datasets"
    if not os.path.exists(Path(root_dir) / COCO_IMAGES):
        raise ValueError(f"{Path(root_dir) / COCO_IMAGES}: please follow the README to set up the datasets "
                         "(or pass --dataset_root)")
    name = f"COCO20k_{args.set}" + ("-nohards" if args.no_hard else "")
    items = []
    for im, anns in coco20k_targets(select_coco20k(root_dir)):
        gt = None
        if not args.no_evaluation:
            gt = extract_gt_coco(anns)
            if gt.shape[0] == 0:
                if args.no_hard:
                    continue
                raise ValueError(f"COCO20k image id {im['id']} has no box that is not a crowd, so CorLoc is undefined "
                                 "for it: pass --no_hard to skip such images (or --no_evaluation)")
        items.append(_Item(str(im["id"]), str(Path(root_dir) / COCO_IMAGES / im["file_name"]), gt,
                           f"COCO_train2014_{int(im['id']):012d}.pth"))
    return name, items


def _eigseg_precomputed(args, items) -> Dict[str, np.ndarray]:
    """--eigenseg --precomputed_eigs_dir: JPEG headers and eigenvector files on reader threads, one kernel call per
    distinct (K, N)."""
    which_matrix = Path(args.precomputed_eigs_dir).name.split("_")[0] if args.which_matrix == "infer" else args.which_matrix
    if which_matrix not in SEGMENT_INDEX:
        raise KeyError(which_matrix)
    row = SEGMENT_INDEX[which_matrix]

    def load(it):
        ev = torch.load(os.path.join(args.precomputed_eigs_dir, it.eig_file), map_location="cpu")
        return jpeg_size(it.path), ev["eigenvectors"].to(torch.float32)

    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        loaded = list(ex.map(load, items))
    groups: Dict[Tuple[int, int], List[int]] = {}
    for j, (_, ev) in enumerate(loaded):
        ev2 = ev.reshape(ev.shape[0], -1)
        groups.setdefault((ev2.shape[0], ev2.shape[1]), []).append(j)
    preds = {}
    dev = torch.device("cuda")
    for (K, N), idx in groups.items():
        evecs = torch.stack([loaded[j][1].reshape(K, N) for j in idx]).to(dev)
        sizes = [loaded[j][0] for j in idx]
        boxes, status = eigseg_boxes(evecs, row, sizes)
        for t, j in enumerate(idx):
            raise_for_status(int(status[t]), items[j].name, N, sizes[t])
            preds[items[j].name] = boxes[t]
    return preds


def _decode_batches(items, batches, load, ahead: int):
    """Decode on reader threads; yields (indices, [uint8 [H, W, 3] numpy]) for each index list of ``batches`` in
    order. At most ``ahead`` batches past the one yielded are decoded or queued, so host memory stays bounded by the
    batches in flight."""
    futs = deque()
    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        nxt = 0
        for k, idx in enumerate(batches):
            while nxt < min(len(batches), k + ahead + 1):
                futs.append([ex.submit(load, items[j]) for j in batches[nxt]])
                nxt += 1
            yield idx, [f.result() for f in futs.popleft()]


def _list_batches(items, batch_size: int, load=None, ahead: int = 2):
    """_decode_batches of batch_size consecutive items in list order, whatever their sizes."""
    batches = [list(range(s, min(s + batch_size, len(items)))) for s in range(0, len(items), batch_size)]
    yield from _decode_batches(items, batches, load or (lambda it: load_rgb(it.path)), ahead)


def _size_batches(sizes: Sequence[Tuple[int, int]], batch_size: int) -> List[List[int]]:
    """Indices grouped by size into batches of at most batch_size: each full batch in the order its last image comes
    in the list, then the partial ones in the order of their first images."""
    full, pending = [], {}
    for j, size in enumerate(sizes):
        group = pending.setdefault(size, [])
        group.append(j)
        if len(group) == batch_size:
            full.append(pending.pop(size))
    return full + list(pending.values())


def _image_batches(items, batch_size: int, load=None, ahead: int = 2):
    """Images of one size per batch; yields (indices, uint8 [B, H, W, 3] numpy). The sizes come from the image
    headers first, so only the batches in flight are decoded however many sizes the list has."""
    with ThreadPoolExecutor(max_workers=io_pipeline.default_workers()) as ex:
        sizes = list(ex.map(lambda it: jpeg_size(it.path), items))
    for idx, imgs in _decode_batches(items, _size_batches(sizes, batch_size), load or (lambda it: load_rgb(it.path)),
                                     ahead):
        batch = np.stack(imgs)
        del imgs   # only the stacked copy stays alive while the caller runs and the next batches decode
        yield idx, batch


def _from_images_ragged(args, items, model, load=None) -> Dict[str, np.ndarray]:
    """LOST and DINO-seg: batch_size images per ragged forward in list order, staged in one page-locked packed buffer;
    the first failing image in list order raises."""
    P = model.patch_size
    ring = io_pipeline.PackedRing(model.device)
    preds = {}
    for idx, imgs in _list_batches(items, max(1, args.batch_size), load):
        slot, host, dims = ring.stage(imgs)
        x = ring.to_device(slot, host)
        if args.dinoseg:
            _, attn, grids = model.forward_last_ragged(x, dims, "k", pad=True, feats=False, cls_attn=True)
            if not 0 <= args.dinoseg_head < model.num_heads:
                raise ValueError(f"--dinoseg_head {args.dinoseg_head} not in [0, {model.num_heads})")
            boxes, status = dinoseg_boxes_ragged(attn, [g[1:] for g in grids], P, args.dinoseg_head)
        else:
            feats, _, grids = model.forward_last_ragged(x, dims, args.which_features, pad=True)
            boxes, _, status = lost_boxes_ragged(feats, [g[1:] for g in grids], dims.tolist(), P, args.k_patches)
        for t, j in enumerate(idx):
            raise_for_status(int(status[t]), items[j].name)
            preds[items[j].name] = boxes[t]
    return preds


def _from_images(args, items, model) -> Dict[str, np.ndarray]:
    if not args.eigenseg:
        return _from_images_ragged(args, items, model)
    # eigen-segmentation keeps batches of one size: the reference crops to whole patches on this route
    # (main.py:220-226), and zero pad rows would change the Laplacian's degrees
    preds = {}
    for idx, imgs in _image_batches(items, max(1, args.batch_size)):
        x = torch.from_numpy(imgs).pin_memory().to(model.device, non_blocking=True)
        B, H, W, _ = x.shape
        feats, _ = model.forward_last(x, args.which_features, pad=False)
        if args.which_matrix == "laplacian":
            _, evecs, _, _ = spectral.laplacian_eigs(feats, 2, normalize=False, threshold_at_zero=True, lapnorm=True)
        else:
            _, evecs, _ = spectral.affinity_eigs(feats, 2, "affinity", normalize=False, threshold_at_zero=False)
        boxes, status = eigseg_boxes(evecs, SEGMENT_INDEX[args.which_matrix], [(H, W)] * B)
        for t, j in enumerate(idx):
            raise_for_status(int(status[t]), items[j].name)
            preds[items[j].name] = boxes[t]
    return preds


def main(argv=None) -> Optional[float]:
    args = parse_args(argv)
    check_supported(args)
    name, items = _dataset_items(args)
    exp_name = experiment_name(args)
    if args.image_path is None:
        args.output_dir = os.path.join(args.output_dir, name)
    exp_dir = Path(args.output_dir) / exp_name
    if args.skip_if_exists and exp_dir.is_dir() and len(list(exp_dir.iterdir())) > 0:
        print(f"Directory already exists and is not empty: {str(exp_dir)}")
        print("Exiting...")
        return None
    os.makedirs(args.output_dir, exist_ok=True)
    print(f"Running LOST on the dataset {name} (exp: {exp_name})")
    print("Args:")
    print(pprint(args.__dict__))

    if args.eigenseg and args.precomputed_eigs_dir is not None:
        preds = _eigseg_precomputed(args, items)
    else:
        model, _, _, _ = vit_mod.get_model(ARCH_MAP[(args.arch, args.patch_size)], checkpoint=args.checkpoint,
                                           seed=args.seed, random_init=args.random_init, precision=args.precision)
        preds = _from_images(args, items, model)

    preds_dict = {it.name: preds[it.name] for it in items}
    if args.image_path is not None:
        print(f"{items[0].name}: {preds_dict[items[0].name].tolist()}")
    gt_dict = {it.name: it.gt for it in items}
    corloc = np.zeros(len(items))
    cnt = 0
    if not args.no_evaluation:
        for i, it in enumerate(items):
            corloc[i] = 1 if corloc_hit(preds_dict[it.name], it.gt) else 0
            cnt += 1
    folder = f"{args.output_dir}/{exp_name}"
    if args.save_predictions:
        os.makedirs(folder, exist_ok=True)
        with open(os.path.join(folder, "preds.pkl"), "wb") as f:
            pickle.dump(preds_dict, f)
        if not args.no_evaluation:
            with open(os.path.join(folder, "gt.pkl"), "wb") as f:
                pickle.dump(gt_dict, f)
        print(f"Predictions saved to {folder}")
    if args.no_evaluation:
        return None
    score = 100 * np.sum(corloc) / cnt
    print(f"corloc: {score:.2f} ({int(np.sum(corloc))}/{cnt})")
    os.makedirs(folder, exist_ok=True)
    result_file = os.path.join(folder, "results.txt")
    with open(result_file, "w") as f:
        f.write("corloc,%.1f,,\n" % score)
    print("File saved at %s" % result_file)
    return float(score)


if __name__ == "__main__":
    main(sys.argv[1:])
