"""Pillow's 8-bit resampler (``Image.resize`` of an RGB image with LANCZOS or BICUBIC, ``reducing_gap=None``) on the device,
bit-exact: the host builds Pillow's fixed-point tables (``precompute_coeffs`` + ``normalize_coeffs_8bpc`` of
libImaging/Resample.c, restated in Python double precision -- Python floats are C doubles, ``math.sin`` is the platform libm),
and ``vcb_resample_u8`` runs one pass per axis in int32.  Images are uint8 [h, w, 3] CUDA tensors (pixels dense, any row stride).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops

LANCZOS, BICUBIC = "lanczos", "bicubic"
PRECISION_BITS = 32 - 8 - 2


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def _bicubic(x: float, a: float = -0.5) -> float:
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


FILTERS = {LANCZOS: (_lanczos, 3.0), BICUBIC: (_bicubic, 2.0)}      # filter, support


def coeffs_8bpc(in_size: int, out_size: int, filt: str):
    """Pillow's tables for resampling one axis of length ``in_size`` to ``out_size`` -> (bounds int32 [out_size, 2] of
    (xmin, n), coeffs int32 [out_size, ksize] with 22 fractional bits, rows zero past n)."""
    if in_size < 1 or out_size < 1:
        raise ValueError(f"resample: sizes must be positive, got {in_size} -> {out_size}")
    f, filter_support = FILTERS[filt]
    scale = in_size / out_size                       # (double)(in1 - in0) / outSize with in0 = 0, in1 = in_size
    filterscale = max(scale, 1.0)
    support = filter_support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), np.int32)
    coeffs = np.zeros((out_size, ksize), np.int32)
    one = 1 << PRECISION_BITS
    for i in range(out_size):
        center = (i + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)                 # int(): C truncation
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [f((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = sum(w)
        if ww != 0.0:
            w = [v / ww for v in w]
        coeffs[i, :n] = [int(-0.5 + v * one) if v < 0 else int(0.5 + v * one) for v in w]
        bounds[i] = (xmin, n)
    return bounds, coeffs


_tables: dict = {}


def _device_tables(in_size: int, out_size: int, filt: str, device):
    """coeffs_8bpc as CUDA tensors, built once per (in_size, out_size, filter, device): a grid reuses a few sizes."""
    key = (in_size, out_size, filt, str(device))
    t = _tables.get(key)
    if t is None:
        b, k = coeffs_8bpc(in_size, out_size, filt)
        t = _tables[key] = (torch.from_numpy(b).to(device), torch.from_numpy(k).to(device))
    return t


def resize(img: torch.Tensor, size, filt: str) -> torch.Tensor:
    """``Image.fromarray(img).resize(size, filt)`` on the device: img uint8 [h, w, 3] CUDA -> uint8 [size[1], size[0], 3].
    The x pass runs first, then the y pass; an axis that keeps its size is not resampled, and ``img`` itself is returned when
    neither changes (Pillow returns a copy)."""
    w_out, h_out = size
    h, w = img.shape[0], img.shape[1]
    if w_out != w:
        out = torch.empty(h, w_out, 3, dtype=torch.uint8, device=img.device)
        ops.resample_u8(img, 0, *_device_tables(w, w_out, filt, img.device), out)
        img = out
    if h_out != h:
        out = torch.empty(h_out, w_out, 3, dtype=torch.uint8, device=img.device)
        ops.resample_u8(img, 1, *_device_tables(h, h_out, filt, img.device), out)
        img = out
    return img


def crop(img: torch.Tensor, box) -> torch.Tensor:
    """``Image.crop(box)`` on the device: a view when the box lies inside the image, else a zero-padded copy."""
    left, top, right, bottom = box
    h, w = img.shape[0], img.shape[1]
    if 0 <= left and 0 <= top and right <= w and bottom <= h:
        return img[top:bottom, left:right]
    out = torch.zeros(bottom - top, right - left, 3, dtype=torch.uint8, device=img.device)
    x0, y0, x1, y1 = max(left, 0), max(top, 0), min(right, w), min(bottom, h)
    if x0 < x1 and y0 < y1:
        out[y0 - top:y1 - top, x0 - left:x1 - left] = img[y0:y1, x0:x1]
    return out


def upload(image, device) -> torch.Tensor:
    """An RGB PIL image -> uint8 [h, w, 3] on ``device``, through a pinned staging buffer."""
    a = np.asarray(image)
    if a.ndim != 3 or a.shape[2] != 3 or a.dtype != np.uint8:
        raise ValueError(f"expected an RGB image, got mode {image.mode}")
    host = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
    host.numpy()[...] = a
    return host.to(device, non_blocking=True)
