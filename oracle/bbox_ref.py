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
