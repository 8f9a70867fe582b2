"""ORACLE (test infrastructure, not product): the reference's box extraction restated with scipy.ndimage.

skimage is not installed here, so skimage.morphology.binary_erosion / binary_dilation (called by the reference's
extract_utils.erode_or_dilate_mask, :115-121) are restated from skimage's documented behaviour: the default footprint is
the 3x3 cross (ndimage.generate_binary_structure(2, 1)), pixels outside the image count as set for erosion
(border_value=True) and as unset for dilation (border_value=False). Parity unpinned by the reference: it ships no
output of these two functions, so the border and footprint rules rest on skimage's documentation, as the DINO ViT and
pymatting restatements rest on theirs."""
from __future__ import annotations

import numpy as np
from scipy import ndimage

CROSS = ndimage.generate_binary_structure(2, 1)


def binary_erosion(image, footprint=None, out=None):
    return ndimage.binary_erosion(image, structure=CROSS if footprint is None else footprint, border_value=True)


def binary_dilation(image, footprint=None, out=None):
    return ndimage.binary_dilation(image, structure=CROSS if footprint is None else footprint, border_value=False)


def erode_or_dilate_mask(x: np.ndarray, r: int = 0, erode: bool = True) -> np.ndarray:
    """extract_utils.py:115-121: r steps; a step whose result is empty is discarded."""
    fn = binary_erosion if erode else binary_dilation
    for _ in range(r):
        x_new = fn(x)
        if x_new.sum() > 0:
            x = x_new
    return x


def extract_bbox(segmap: np.ndarray, image_id, P: int, num_erode: int, num_dilate: int, skip_bg_index: bool) -> dict:
    """_extract_bbox (extract.py:429-470) on an in-memory label map, with the same element types."""
    outputs = {"bboxes": [], "bboxes_original_resolution": [], "segment_indices": [], "id": image_id,
               "format": "(xmin, ymin, xmax, ymax)"}
    for segment_index in sorted(np.unique(segmap).tolist()):
        if (not skip_bg_index) or (segment_index > 0):
            binary_mask = segmap == segment_index
            binary_mask = erode_or_dilate_mask(binary_mask, r=num_erode, erode=True)
            binary_mask = erode_or_dilate_mask(binary_mask, r=num_dilate, erode=False)
            mask = np.where(binary_mask == 1)
            ymin, ymax = min(mask[0]), max(mask[0]) + 1
            xmin, xmax = min(mask[1]), max(mask[1]) + 1
            bbox = [xmin, ymin, xmax, ymax]
            outputs["segment_indices"].append(segment_index)
            outputs["bboxes"].append(bbox)
            outputs["bboxes_original_resolution"].append([x * P for x in bbox])
    return outputs


def edge_maps(H: int, W: int, seed: int = 0) -> dict:
    """Hand-built label maps at an H x W grid for the morphology's edges (name -> uint8 map): every one of the 256 values
    at once, only 0, only 255, 1-pixel lines, a 0 / 255 checkerboard (every pixel isolated: erosion empties it at step
    1), squares of sides 1, 3, 5, ... (side 2s - 1 empties at erosion step s), segments touching each border and
    corner (where erosion's outside-is-set and dilation's outside-is-unset rules differ), random rectangles."""
    g = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    maps = {"all_values": np.resize(g.permutation(256), H * W).reshape(H, W),
            "zeros": np.zeros((H, W)), "ones255": np.full((H, W), 255),
            "checker": ((y + x) % 2) * 255}
    lines = np.zeros((H, W))
    lines[y % 4 == 1] = 1 + (y[y % 4 == 1] // 4) % 100
    lines[x % 5 == 2] = 101 + (x[x % 5 == 2] // 5) % 100
    maps["lines"] = lines
    sq = np.full((H, W), 7)
    r0, c0, v = int(H > 2), int(W > 2), 1      # off the border where there is room: clipped squares on a strip
    for side in range(1, 40, 2):
        if c0 >= W:
            r0, c0 = r0 + side + 1, int(W > 2)
        if r0 >= H:
            break
        sq[r0:r0 + side, c0:c0 + side] = 10 + v
        c0 += side + 1
        v += 1
    maps["squares"] = sq
    border = np.full((H, W), 50)
    border[:, : max(1, W // 6)] = 51
    border[:, W - max(1, W // 7):] = 52
    border[: max(1, H // 5)] = 53
    border[H - max(1, H // 8):] = 54
    border[0, 0], border[0, W - 1], border[H - 1, 0], border[H - 1, W - 1] = 60, 61, 62, 63
    border[H // 2, W // 2] = 64
    maps["border"] = border
    rects = np.zeros((H, W))
    for v in g.choice(np.arange(1, 256), size=min(40, H * W), replace=False):
        r, c = g.integers(0, H), g.integers(0, W)
        rects[r:r + g.integers(1, max(2, H // 2)), c:c + g.integers(1, max(2, W // 2))] = v
    maps["rects"] = rects
    return {k: np.ascontiguousarray(m, dtype=np.uint8) for k, m in maps.items()}
