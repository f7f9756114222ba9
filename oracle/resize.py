"""A plain restatement of Pillow's bicubic resize of an 8-bit image (Image.resize(size) with its default filter, for
modes "RGB" and "L") -- the reference csrc/resize.cu is tested against.

    out = resize_u8(planes, width, height)         # uint8 (..., H, W) -> (..., height, width)
    bounds, coeffs = plan(in_size, out_size)       # one axis: (out, 2) int32 [first tap, taps], (out, ksize) int32

Per axis, with scale = in / out and filterscale = max(scale, 1), output index i has
    center = (i + 0.5) * scale,  support = 2 * filterscale,
    first  = max(int(center - support + 0.5), 0),  last = min(int(center + support + 0.5), in),
and its taps j = 0 .. last - first weigh input first + j by bicubic((j + first - center + 0.5) * (1 / filterscale)),
the Keys cubic with a = -0.5: (1.5 t - 2.5) t t + 1 for |t| < 1, (((t - 5) t + 8) t - 4) * -0.5 for |t| < 2, else 0.
Each weight is divided by the taps' double sum (left to right; skipped when the sum is 0) and made fixed-point at 22
bits, rounding half away from zero: int(w * 2^22 +- 0.5), truncated.  A pass sums pixel * weight in int32 from 2^21
and writes clamp(sum >> 22, 0, 255).  The horizontal pass runs first into a uint8 intermediate; the vertical pass
reads it.  An axis whose size does not change is not resampled.

Every step is IEEE double or integer arithmetic in a fixed order, so the device gives the same bytes when it does the
same operations without contraction.
"""
from __future__ import annotations

import math

import numpy as np

PRECISION_BITS = 22
SUPPORT = 2.0


def bicubic(t: float) -> float:
    t = abs(t)
    if t < 1.0:
        return (1.5 * t - 2.5) * t * t + 1
    if t < 2.0:
        return (((t - 5) * t + 8) * t - 4) * -0.5
    return 0.0


def ksize(in_size: int, out_size: int) -> int:
    """Taps per output index: the table's row length."""
    filterscale = max(float(in_size) / out_size, 1.0)
    return int(math.ceil(SUPPORT * filterscale)) * 2 + 1


def plan(in_size: int, out_size: int) -> tuple:
    """(bounds (out, 2) int32 of [first input, taps], coeffs (out, ksize) int32 fixed-point weights, 0 past the taps)
    of one axis."""
    if in_size < 1 or out_size < 1:
        raise ValueError(f"sizes must be positive, got {in_size} -> {out_size}")
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = SUPPORT * filterscale
    ss = 1.0 / filterscale
    K = ksize(in_size, out_size)
    bounds = np.zeros((out_size, 2), np.int32)
    coeffs = np.zeros((out_size, K), np.int32)
    for i in range(out_size):
        center = (i + 0.5) * scale
        first = max(int(center - support + 0.5), 0)
        taps = min(int(center + support + 0.5), in_size) - first
        w = [bicubic((j + first - center + 0.5) * ss) for j in range(taps)]
        total = 0.0
        for v in w:
            total += v
        if total != 0.0:
            w = [v / total for v in w]
        for j, v in enumerate(w):
            coeffs[i, j] = int(v * (1 << PRECISION_BITS) + (-0.5 if v < 0 else 0.5))
        bounds[i] = first, taps
    return bounds, coeffs


def _pass(src: np.ndarray, bounds: np.ndarray, coeffs: np.ndarray) -> np.ndarray:
    """Resamples the last axis of int64 `src` by one axis plan -> uint8."""
    n_out, K = coeffs.shape
    idx = np.minimum(bounds[:, :1] + np.arange(K)[None, :], src.shape[-1] - 1)       # (out, K); weight 0 past taps
    acc = (src[..., idx] * coeffs.astype(np.int64)).sum(-1) + (1 << (PRECISION_BITS - 1))
    assert np.abs(acc).max(initial=0) < 2**31     # the device's int32 accumulator holds every partial sum too
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize_u8(planes: np.ndarray, width: int, height: int) -> np.ndarray:
    """uint8 (..., H, W) planes -> (..., height, width): each plane as Pillow resizes an "L" image (and each channel of
    an "RGB" image) to (width, height)."""
    a = np.asarray(planes)
    if a.dtype != np.uint8 or a.ndim < 2:
        raise ValueError(f"planes must be uint8 (..., H, W), got {a.dtype} {a.shape}")
    H, W = a.shape[-2:]
    out = a
    if width != W:
        out = _pass(out.astype(np.int64), *plan(W, width))
    if height != H:
        out = np.swapaxes(_pass(np.swapaxes(out, -1, -2).astype(np.int64), *plan(H, height)), -1, -2)
    return np.ascontiguousarray(out)
