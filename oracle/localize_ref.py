"""ORACLE (test infrastructure, not product): numpy / scipy restatement of the reference's object localization
(object-localization/object_discovery.py, datasets.py, main.py) and the last-block ViT outputs it hooks.

Component labels come from scipy.ndimage.label (numbered by the raster position of each component's first pixel, as
skimage.measure.label numbers them too): 8-connectivity (ones((3, 3))) where the reference calls skimage's label with
its default connectivity=ndim, the default cross where it calls scipy's. LOST orders patches by ascending degree with
ties by patch index (the reference's unstable argsort leaves ties unspecified)."""
from __future__ import annotations

import math

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


def lost_expand(rows, N, k_patches=100, chunk=1024):
    """lost's seed, similars and M for A [N, N] given as rows(idx) -> fp32 [len(idx), N], so that a device A is read in
    row chunks. The seed and potentials follow lost_order; M sums the similar rows in fp32 one after the other in
    potentials order, which is the kernel's order (the reference's torch.sum may round differently: sum_decided)."""
    deg = np.empty(N, dtype=np.int64)
    for r0 in range(0, N, chunk):
        idx = np.arange(r0, min(N, r0 + chunk))
        pos = rows(idx) > 0
        pos[np.arange(idx.size), idx] = False
        deg[idx] = pos.sum(1)
    order = np.lexsort((np.arange(N), deg))
    seed = int(order[0])
    pot = order[:k_patches]
    sim = pot[rows(np.asarray([seed]))[0][pot] > 0]
    M = np.zeros(N, dtype=np.float32)
    for c0 in range(0, sim.size, chunk):
        for r in rows(sim[c0:c0 + chunk]):
            M += r
    return seed, sim, M


def detect_box(M, seed, grid, size, P):
    """detect_box on M [N] -> (int64 [4], status): status 2 (boxes zero) when the seed is in the background."""
    gh, gw = grid
    lab, _ = scipy.ndimage.label(np.asarray(M).reshape(gh, gw) > 0)
    cc = lab.ravel()[seed]
    if cc == 0:
        return np.zeros(4, dtype=np.int64), 2
    ys, xs = np.where(lab == cc)
    H, W = size
    return np.asarray([P * xs.min(), P * ys.min(), min(P * (xs.max() + 1), W), min(P * (ys.max() + 1), H)],
                      dtype=np.int64), 0


def lost_box(A, grid, size, P, k_patches=100):
    """lost + detect_box on A [N, N] fp32 (F F^T), grid (gh, gw), un-padded size (H, W) -> (int64 [4], seed)."""
    A = np.asarray(A, dtype=np.float32)
    seed, _, M = lost_expand(lambda idx: A[idx], A.shape[0], k_patches)
    box, status = detect_box(M, seed, grid, size, P)
    if status:
        raise ValueError("The seed is in the background component.")
    return box, seed


def sum_decided(rows):
    """(float64 sum over axis 0 of rows [n, N], cells whose sign every fp32 summation order gets right). Any order of
    fp32 additions is within gamma_(n-1) sum|a| of the exact sum (Higham, Accuracy and Stability, 4.2), u = 2^-24;
    gamma_n is used so that the float64 sum's own rounding cannot decide a cell either."""
    a = np.asarray(rows, dtype=np.float64)
    n, u = a.shape[0], 2.0 ** -24
    m64 = a.sum(0)
    return m64, np.abs(m64) > n * u / (1 - n * u) * np.abs(a).sum(0)


def dinoseg_kept(attn_row, total="torch"):
    """The kept mask of dino_seg for one head: torch CPU sort (ties by index), /sum, cumsum, > 1 - 0.6. total="torch"
    divides by torch's float sum as the reference does; "fp64" by the exactly rounded sum, as the kernel does."""
    a = torch.as_tensor(np.asarray(attn_row, dtype=np.float32))[None]
    val, idx = torch.sort(a, stable=True)
    if total == "torch":
        val = val / torch.sum(val, dim=1, keepdim=True)
    else:
        val = val / torch.tensor(np.float32(math.fsum(np.asarray(attn_row, dtype=np.float64))))
    th = torch.cumsum(val, dim=1) > (1 - 0.6)
    kept = torch.zeros_like(th)
    kept[0, idx[0]] = th[0]
    return kept[0].numpy()


def dinoseg_select(kept, grid, P):
    """dino_seg's component choice on a kept mask [N] -> (int64 [4], status): status 3 (boxes zero) when the selected
    label has no cell."""
    gh, gw = grid
    lab, _ = scipy.ndimage.label(np.asarray(kept).reshape(gh, gw).astype(np.float32))
    sizes = np.bincount(lab.ravel())[:np.max(lab)]             # [np.sum(lab == c) for c in range(np.max(lab))]
    c = int(np.argmax(sizes[1:])) + 1 if len(sizes) > 1 else 0
    ys, xs = np.where(lab == c)
    if ys.size == 0:
        return np.zeros(4, dtype=np.int64), 3
    return np.asarray([xs.min() * P, ys.min() * P, (xs.max() + 1) * P, (ys.max() + 1) * P], dtype=np.int64), 0


def dinoseg_box(attn_row, grid, P):
    """dino_seg's component choice on one head's CLS attention [N] -> int64 [4]; ValueError on an empty selection."""
    box, status = dinoseg_select(dinoseg_kept(attn_row), grid, P)
    if status:
        raise ValueError("DINO-seg selected an empty component")
    return box


# Dyadic DINO-seg rows: integer multiples of 2^-25 that sum to 2^25 units, so that the normalising sum is exactly 1 and
# every cumulative mass is exact in fp32 (below 0.5 any multiple of 2^-25 is; from 0.5 on, the prefixes are even).
DYADIC_UNIT = 2.0 ** -25
THRESHOLD_UNITS = 13421773          # fl32(0.4) = 0x3ECCCCCD = 13421773 * 2^-25, the threshold dino_seg compares with


def dyadic_row(kept, tie_cell=None):
    """Integer units [N] (sum 2^25) whose dino_seg kept mask is `kept` [N] bool: the non-kept cells hold exactly
    fl32(0.4), most of them 0 (runs of exact zeros), so the last non-kept cell in sorted order ends on the threshold
    itself and is not kept. The lowest kept value is the only odd one among the kept and sits at the smallest kept
    index. tie_cell: a non-kept cell of smaller index that gets that same lowest kept value, so the two straddle the
    threshold and only the order of ties by index decides between them. ValueError when no such row exists (fewer than
    2 or all cells kept, too few non-kept cells for the mass) or when torch's float sum or cumsum of it is inexact."""
    kept = np.asarray(kept, dtype=bool).ravel()
    N, k = kept.size, int(kept.sum())
    if not 2 <= k < N:
        raise ValueError(f"no dyadic row keeps {k} of {N} cells")
    units = np.zeros(N, dtype=np.int64)
    kidx, nidx = np.flatnonzero(kept), np.flatnonzero(~kept)
    mass = 2 ** 25 - THRESHOLD_UNITS
    a = mass // (2 * k)
    j = min((mass - 2 * a * k + 1) // 2, k - 1)               # other kept cells: 2a, j of them 2a + 2
    units[kidx[1:]] = 2 * a
    units[kidx[k - j:]] += 2 if j else 0
    low = mass - units[kidx[1:]].sum()
    assert low % 2 == 1 and 0 < low < units[kidx[1:]].min(initial=low + 1)
    units[kidx[0]] = low
    rest = THRESHOLD_UNITS
    if tie_cell is not None:
        assert not kept[tie_cell] and tie_cell < kidx[0]
        units[tie_cell] = low
        rest -= low
        nidx = nidx[nidx != tie_cell]
    w = low - 1                                               # the largest non-kept value below the lowest kept one
    full, r = divmod(rest, w)
    if full + (r > 0) > nidx.size:
        raise ValueError("not enough non-kept cells for the mass below the threshold")
    if full:
        units[nidx[nidx.size - full:]] = w
    if r:
        units[nidx[0]] = r
    if not dyadic_exact(units):
        raise ValueError("torch's float sum or cumsum of this row is not exact")
    return units


def dyadic_exact(units):
    """True when the fp32 row units * 2^-25 holds the units exactly, and its float64 sum, torch's CPU float sum of the
    sorted row and every prefix of torch's cumsum of it equal the integer fractions."""
    row = (np.asarray(units) * DYADIC_UNIT).astype(np.float32)
    s = torch.sort(torch.from_numpy(row), stable=True)[0]
    prefix = np.cumsum(np.sort(units)) * DYADIC_UNIT
    return bool((row.astype(np.float64) / DYADIC_UNIT == units).all() and math.fsum(row) == 1.0
                and torch.sum(s).item() == 1.0 and (torch.cumsum(s, 0).numpy() == prefix).all())


def cc_patterns(gh, gw):
    """Masks [gh, gw] bool where a connected-components routine can go wrong, by name (random masks rarely produce
    them): all / none set; the first N / 2 and N / 2 + 1 cells in raster order; cells on both ends of a row and on
    opposite ends of consecutive rows (raster neighbours that are not grid neighbours); a U whose arms join only in the
    bottom row; a serpentine; a checkerboard (one component under 8-connectivity, singletons under 4); two equal largest
    blocks, alone and followed by a smaller last-numbered component; a small component numbered before a large one;
    isolated cells at every other row and column (4096 roots at 128 x 128)."""
    N = gh * gw
    r, c = np.indices((gh, gw))
    flat = np.arange(N).reshape(gh, gw)
    out = {"all": np.ones((gh, gw), bool), "none": np.zeros((gh, gw), bool),
           "half": flat < N // 2, "half_plus_one": flat < N // 2 + 1,
           "row_ends": (r % 2 == 0) & ((c == 0) | (c == gw - 1)),
           "row_wrap": ((r % 2 == 0) & (c == gw - 1)) | ((r % 2 == 1) & (c == 0)),
           "u": (c == 0) | (c == gw - 1) | (r == gh - 1),
           "serpentine": (r % 2 == 0) | ((r % 4 == 1) & (c == gw - 1)) | ((r % 4 == 3) & (c == 0)),
           "checkerboard": (r + c) % 2 == 0,
           "dots": (r % 2 == 0) & (c % 2 == 0)}
    bh, bw = max(1, gh // 4), max(1, gw // 4)
    twin = np.zeros((gh, gw), bool)
    twin[:bh, :bw] = True
    twin[gh - bh:, gw - bw:] = True
    out["twin"] = twin
    small = twin.copy()
    small[:bh, :bw] = False
    small[0, 0] = True
    out["small_then_large"] = small
    if bh >= 2 and gw - bw - 2 >= 0:                # a single cell in the last row, left of the second block
        third = twin.copy()
        third[gh - 1, gw - bw - 2] = True
        out["twin_then_small"] = third
    return out


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


def cls_attention_bound(qkv_f16: torch.Tensor, heads: int):
    """(float64 softmax [B, heads, T - 1], per-element bound on |fp32 kernel - float64|) for an fp16 qkv [B, T, 3d].
    A 64-term fp32 fma score is within e_j = gamma_64 sum|q k| / 8 of the exact one; subtracting the max rounds by
    u (|s_j - max| + 2 max e); expf is within 2 ulp; the fp32 sum of T positive terms within gamma_T; the division u.
    The errors in the exponents enter numerator and denominator, hence exp(D_j + max D) - 1; an underflowed term may be
    off by 2^-149 absolutely."""
    u = 2.0 ** -24
    q = qkv_f16.double().cpu()
    B, T, d3 = q.shape
    d = d3 // 3
    q0 = q[:, 0, :d].reshape(B, heads, 1, 64)
    k = q[:, :, d:2 * d].reshape(B, T, heads, 64).permute(0, 2, 1, 3)
    s = (q0 * k).sum(-1) / 8
    e = 64 * u / (1 - 64 * u) * (q0.abs() * k.abs()).sum(-1) / 8
    D = e + u * ((s - s.amax(-1, keepdim=True)).abs() + 2 * e.amax(-1, keepdim=True))
    rel = torch.expm1(D + D.amax(-1, keepdim=True) + 2 * 2.0 ** -22 + T * u / (1 - T * u) + 2 * u)
    p = torch.softmax(s, -1)
    return p[..., 1:], (rel * p + 2.0 ** -148)[..., 1:]
