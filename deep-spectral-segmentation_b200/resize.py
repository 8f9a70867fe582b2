"""Pillow's ``Image.resize((W_out, H_out), Image.BILINEAR)`` of RGB images, bit for bit, on the device.

The reference builds the colour affinities from the whole image resized with PIL (extract/extract.py:199-204). Pillow's
bilinear is not F.interpolate: per axis it

  * widens the triangle filter's support by the scale factor when it downscales (so it antialiases),
  * normalises each output pixel's weights to sum 1 and rounds them to fixed point with 22 fractional bits,
  * runs a horizontal pass, then a vertical pass over the horizontal pass's rounded, clipped uint8 image.

``coeffs`` restates the window and weight arithmetic on the host in double precision (Python floats), operation by
operation; ``resize_host`` is the integer two-pass resize in numpy (the reference for the tests); ``resize`` runs the
same arithmetic in csrc/resize.cu for a batch of images of one size already on the device. An axis whose output size
equals its input size gets the weights {1, 0}, which reproduce every value exactly, so the device kernel always runs
both passes where Pillow skips one."""
from __future__ import annotations

from functools import lru_cache
from typing import Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

PRECISION_BITS = 22           # 32 - 8 - 2: fixed-point fraction of the weights
KINDS = {"u8": 0, "f32": 1}   # DSS_RESIZE_U8 / DSS_RESIZE_UNIT_F32


def _triangle(x: float) -> float:
    if x < 0.0:
        x = -x
    if x < 1.0:
        return 1.0 - x
    return 0.0


@lru_cache(maxsize=1024)
def _coeffs(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    if in_size <= 0 or out_size <= 0:
        raise ValueError(f"resize: sizes must be positive (input {in_size}, output {out_size})")
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    taps = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), np.int32)
    weights = np.zeros((out_size, taps), np.int32)
    one = float(1 << PRECISION_BITS)
    for o in range(out_size):
        center = (o + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)        # int() truncates toward zero, as the C cast does
        hi = min(int(center + support + 0.5), in_size) - lo
        w = [_triangle((x + lo - center + 0.5) * ss) for x in range(hi)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        weights[o, :hi] = [int(-0.5 + v * one) if v < 0 else int(0.5 + v * one) for v in w]
        bounds[o] = (lo, hi)
    bounds.setflags(write=False)
    weights.setflags(write=False)
    return bounds, weights


def coeffs(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    """Window bounds [out_size, 2] int32 {first input index, count} and fixed-point weights [out_size, taps] int32
    (zero past each count) of one axis."""
    return _coeffs(int(in_size), int(out_size))


def _clip8(acc: np.ndarray) -> np.ndarray:
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)   # acc >= 0: bilinear weights are never negative


def _pass(img: np.ndarray, bounds: np.ndarray, weights: np.ndarray, axis: int) -> np.ndarray:
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((len(bounds),) + src.shape[1:], np.uint8)
    for o, (lo, n) in enumerate(bounds.tolist()):
        acc = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for t in range(n):
            acc += src[lo + t] * int(weights[o, t])
        out[o] = _clip8(acc)
    return np.moveaxis(out, 0, axis)


def resize_host(img: np.ndarray, W_out: int, H_out: int) -> np.ndarray:
    """uint8 [H, W, C] -> uint8 [H_out, W_out, C]: the fixed-point two-pass resize in numpy (horizontal, then vertical)."""
    H, W = img.shape[:2]
    tmp = _pass(img, *coeffs(W, W_out), axis=1)
    return _pass(tmp, *coeffs(H, H_out), axis=0)


@torch.no_grad()
def resize(images: Union[torch.Tensor, Sequence[torch.Tensor]], H_out: int, W_out: int, kind: str = "u8"
           ) -> torch.Tensor:
    """Device batch of uint8 RGB images [B, H, W, 3] (or a list of [H, W, 3] CUDA tensors of one size) ->
    [B, H_out * W_out, 3]: uint8 pixels for ``kind='u8'``, or for ``kind='f32'`` fp32 equal to numpy's
    ``(pixels / 255.0).astype(np.float32)``. Downscaling (or keeping a size) only."""
    if kind not in KINDS:
        raise ValueError(f"resize: unknown output kind {kind!r} (one of {sorted(KINDS)})")
    if not isinstance(images, torch.Tensor):
        images = list(images)
        if not images:
            raise ValueError("resize: no images")
        for j, im in enumerate(images):
            if im.dim() != 3 or im.shape[-1] != 3:
                raise ValueError(f"resize: image {j} is not a 3-channel HWC image (shape {tuple(im.shape)})")
            if im.shape != images[0].shape:
                raise ValueError(f"resize: image {j} is {tuple(im.shape[:2])}, image 0 is {tuple(images[0].shape[:2])}: "
                                 "one call resizes images of one size")
        images = torch.stack(images)
    if images.dim() != 4 or images.shape[-1] != 3:
        raise ValueError(f"resize: expected 3-channel images [B, H, W, 3], got shape {tuple(images.shape)}")
    if images.dtype != torch.uint8:
        raise ValueError(f"resize: expected uint8 pixels, got {images.dtype}")
    B, H, W, _ = images.shape
    H_out, W_out = int(H_out), int(W_out)
    if not (0 < H_out <= H and 0 < W_out <= W):
        raise ValueError(f"resize: output {H_out} x {W_out} must be non-empty and no larger than the input {H} x {W}")
    _lib.require_cuda(images, "images")
    by, wy = coeffs(H, H_out)
    bx, wx = coeffs(W, W_out)
    lib = _lib.load()
    x = images.contiguous()
    dev = x.device
    out = torch.empty(B, H_out * W_out, 3, dtype=torch.uint8 if kind == "u8" else torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = torch.empty(max(256, int(lib.dss_resize_workspace_bytes(H_out, W_out, wy.shape[1], wx.shape[1]))),
                         dtype=torch.uint8, device=dev)
        _lib.check(lib.dss_resize_bilinear(x.data_ptr(), B, H, W, H_out, W_out, by.ctypes.data, wy.ctypes.data,
                                           wy.shape[1], bx.ctypes.data, wx.ctypes.data, wx.shape[1], KINDS[kind],
                                           out.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)),
                   "dss_resize_bilinear")
    return out
