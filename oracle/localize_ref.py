"""ORACLE (test infrastructure, not product): numpy / scipy restatement of the reference's object localization
(object-localization/object_discovery.py, datasets.py, main.py) and the last-block ViT outputs it hooks.

Component labels come from scipy.ndimage.label (numbered by the raster position of each component's first pixel, as
skimage.measure.label numbers them too): 8-connectivity (ones((3, 3))) where the reference calls skimage's label with
its default connectivity=ndim, the default cross where it calls scipy's. LOST orders patches by ascending degree with
ties by patch index (the reference's unstable argsort leaves ties unspecified)."""
from __future__ import annotations

import numpy as np
import scipy.ndimage
import torch
import torch.nn.functional as F

from .dino_vit import IMAGENET_MEAN, IMAGENET_STD

EIGHT = np.ones((3, 3), dtype=int)


def eigseg_grid(N, H, W):
    """(P, H_lr, W_lr) of get_bbox_from_patch_mask's four cases, or None."""
    if (H // 8) * (W // 8) == N:
        return 8, H // 8, W // 8
    if (H // 16) * (W // 16) == N:
        return 16, H // 16, W // 16
    if 4 * (H // 16) * (W // 16) == N:
        return 8, 2 * (H // 16), 2 * (W // 16)
    if 16 * (H // 32) * (W // 32) == N:
        return 8, 4 * (H // 32), 4 * (W // 32)
    return None


def eigseg_box(v, H, W):
    """get_bbox_from_patch_mask(v > 0, (3, H, W)) -> int64 [4]; ValueError when no grid fits."""
    v = np.asarray(v, dtype=np.float32).reshape(-1)
    g = eigseg_grid(v.size, H, W)
    if g is None:
        raise ValueError(f"no patch grid for {(H, W)} with {v.size} cells")
    P, h, w = g
    m = (v > 0).reshape(h, w)
    s = int(m.sum())
    if 0.5 < m.mean() < 1.0 or s == 0:
        m = ~m
    lab, _ = scipy.ndimage.label(m, structure=EIGHT)
    c = int(np.argmax(np.bincount(lab.ravel())[1:])) + 1
    ys, xs = np.where(lab == c)
    return np.asarray([P * xs.min(), P * ys.min(), min(P * (xs.max() + 1), W), min(P * (ys.max() + 1), H)],
                      dtype=np.int64)


def lost_order(A):
    """Patches by ascending degree #{j != i : A_ij > 0}, ties by index."""
    B = np.array(A, dtype=np.float32, copy=True)
    np.fill_diagonal(B, 0)
    deg = (B > 0).sum(1)
    return np.lexsort((np.arange(len(deg)), deg))


def lost_box(A, grid, size, P, k_patches=100):
    """lost + detect_box on A [N, N] fp32 (F F^T), grid (gh, gw), un-padded size (H, W) -> (int64 [4], seed)."""
    A = np.asarray(A, dtype=np.float32)
    order = lost_order(A)
    seed = int(order[0])
    pot = order[:k_patches]
    sim = pot[A[seed, pot] > 0]
    M = np.zeros(A.shape[1], dtype=np.float32)
    for s in sim:                      # fp32, in potentials order
        M = (M + A[s]).astype(np.float32)
    gh, gw = grid
    lab, _ = scipy.ndimage.label(M.reshape(gh, gw) > 0)
    cc = lab[np.unravel_index(seed, (gh, gw))]
    if cc == 0:
        raise ValueError("The seed is in the background component.")
    ys, xs = np.where(lab == cc)
    H, W = size
    return np.asarray([P * xs.min(), P * ys.min(), min(P * (xs.max() + 1), W), min(P * (ys.max() + 1), H)],
                      dtype=np.int64), seed


def dinoseg_kept(attn_row):
    """The kept mask of dino_seg for one head: torch CPU sort (ties by index), /sum, cumsum, > 1 - 0.6."""
    a = torch.as_tensor(np.asarray(attn_row, dtype=np.float32))[None]
    val, idx = torch.sort(a, stable=True)
    val = val / torch.sum(val, dim=1, keepdim=True)
    th = torch.cumsum(val, dim=1) > (1 - 0.6)
    kept = torch.zeros_like(th)
    kept[0, idx[0]] = th[0]
    return kept[0].numpy()


def dinoseg_box(attn_row, grid, P):
    """dino_seg's component choice on one head's CLS attention [N] -> int64 [4]; ValueError on an empty selection."""
    gh, gw = grid
    lab, _ = scipy.ndimage.label(dinoseg_kept(attn_row).reshape(gh, gw).astype(np.float32))
    sizes = [np.sum(lab == c) for c in range(np.max(lab))]
    c = int(np.argmax(sizes[1:])) + 1 if len(sizes) > 1 else 0
    ys, xs = np.where(lab == c)
    if ys.size == 0:
        raise ValueError("DINO-seg selected an empty component")
    return np.asarray([xs.min() * P, ys.min() * P, (xs.max() + 1) * P, (ys.max() + 1) * P], dtype=np.int64)


def extract_gt_voc(target, remove_hards=False):
    """extract_gt_VOC on a VOCDetection target dict -> int64 [n, 4]."""
    out = []
    for o in target["annotation"]["object"]:
        if remove_hards and (o["truncated"] == "1" or o["difficult"] == "1"):
            continue
        b = o["bndbox"]
        out.append([int(b["xmin"]) - 1, int(b["ymin"]) - 1, int(b["xmax"]), int(b["ymax"])])
    return np.asarray(out)


def iou_float64(box, gts):
    """The same formula in float64 (what a naive restatement would compute; used to find boundary cases)."""
    box, gts = np.asarray(box, np.float64), np.asarray(gts, np.float64).reshape(-1, 4)
    iw = np.clip(np.minimum(box[2], gts[:, 2]) - np.maximum(box[0], gts[:, 0]), 0, None)
    ih = np.clip(np.minimum(box[3], gts[:, 3]) - np.maximum(box[1], gts[:, 1]), 0, None)
    inter = iw * ih
    union = (box[2] - box[0]) * (box[3] - box[1] + 1e-7) + (gts[:, 2] - gts[:, 0]) * (gts[:, 3] - gts[:, 1] + 1e-7) \
        - inter + 1e-7
    return inter / union


# ------------------------------------------------------------------------------------------------ ViT
def preprocess_pad(img_hwc_u8: torch.Tensor, patch: int) -> torch.Tensor:
    """uint8 RGB (H, W, 3) -> (1, 3, ceil(H/P) P, ceil(W/P) P) fp32: ToTensor + Normalize, zeros outside the image
    (object-localization/main.py:227-235)."""
    H, W, _ = img_hwc_u8.shape
    x = img_hwc_u8.permute(2, 0, 1).to(torch.float32).div(255.0)
    x = (x - torch.tensor(IMAGENET_MEAN).view(3, 1, 1)) / torch.tensor(IMAGENET_STD).view(3, 1, 1)
    Hp, Wp = -(-H // patch) * patch, -(-W // patch) * patch
    out = torch.zeros(1, 3, Hp, Wp)
    out[0, :, :H, :W] = x
    return out


@torch.no_grad()
def last_outputs(model, images: torch.Tensor, which: str = "k"):
    """For the oracle DinoViT: (the `which` third of the last block's qkv, CLS row dropped [B, N, d],
    get_last_selfattention(images)[:, :, 0, 1:] [B, heads, N]) -- the qkv hook and attention of main.py:283-322."""
    d, nh = model.cfg.dim, model.cfg.heads
    x = model.prepare_tokens(images)
    for blk in model.blocks[:-1]:
        x = blk(x)
    blk = model.blocks[-1]
    qkv = blk.attn.qkv(blk.norm1(x))
    B, T, _ = qkv.shape
    t = {"q": 0, "k": 1, "v": 2}[which]
    feats = qkv[:, 1:, t * d:(t + 1) * d].contiguous()
    q = qkv[..., :d].reshape(B, T, nh, 64).permute(0, 2, 1, 3)
    k = qkv[..., d:2 * d].reshape(B, T, nh, 64).permute(0, 2, 1, 3)
    attn = ((q @ k.transpose(-2, -1)) * blk.attn.scale).softmax(dim=-1)
    return feats, attn[:, :, 0, 1:].contiguous()


def cls_attention_from_qkv(qkv_f16: torch.Tensor, heads: int) -> torch.Tensor:
    """fp32 softmax(q_0 k_j / 8)[1:] of an fp16 qkv [B, T, 3d] (what dss_op_cls_attention computes)."""
    q = qkv_f16.float()
    B, T, d3 = q.shape
    d = d3 // 3
    q0 = q[:, 0, :d].reshape(B, heads, 1, 64)
    k = q[:, :, d:2 * d].reshape(B, T, heads, 64).permute(0, 2, 1, 3)
    s = (q0.double() @ k.double().transpose(-2, -1))[:, :, 0] / 8.0
    return F.softmax(s, dim=-1)[:, :, 1:]
