"""Frame sequences for the H.264 stream encoder's P pictures (tests/h264_stream_oracle.py, gab200_h264_encode_stream):
identical frames, content shifted by known whole-sample amounts, pans whose vectors reach outside the picture on
every side, a scene cut, noise, odd padded sizes and a GOP long enough for frame_num to wrap.

    for name, frames, qp, gop in sequences(): ...      # frames (K, H, W, 3) uint8
"""
from __future__ import annotations

import numpy as np

from tests import h264_corpus as hc


def shifted(img, dx: int, dy: int):
    """img moved right by dx and down by dy samples, the uncovered side filled by edge replication -- what a vector
    read at clamped coordinates predicts exactly."""
    h, w, _ = img.shape
    p = max(abs(dx), abs(dy))
    big = np.pad(img, ((p, p), (p, p), (0, 0)), mode="edge")
    return np.ascontiguousarray(big[p - dy:p - dy + h, p - dx:p - dx + w])


def static(w, h, n, seed=1):
    return np.stack([hc.textured(w, h, seed=seed)] * n)


def drift(w, h, steps, seed=4):
    """A textured frame moved by each (dx, dy) of steps in turn."""
    f = [hc.textured(w, h, seed=seed)]
    for dx, dy in steps:
        f.append(shifted(f[-1], dx, dy))
    return np.stack(f)


def pan(w, h):
    """Moves toward every side in turn: edge macroblocks' vectors point outside the picture on all four sides."""
    return drift(w, h, [(3, 2), (-5, -4), (2, 5), (0, -6), (16, -16), (-16, 16)], seed=6)


def scene_cut(w, h):
    a, b = hc.textured(w, h, seed=2), hc.stripes(w, h, True)
    return np.stack([a, shifted(a, 1, 0), b, shifted(b, 0, 1), hc.gradient(w, h)])


def noisy(w, h, n=4):
    return np.stack([hc.noise(w, h, seed=20 + k) for k in range(n)])


def soft(w, h, n=4):
    """Low-amplitude noise over a drifting texture: small residual levels in most blocks."""
    base = drift(w, h, [(1, 0)] * (n - 1), seed=8).astype(np.int64)
    rng = np.random.default_rng(9)
    return (base + rng.integers(-6, 7, base.shape)).clip(0, 255).astype(np.uint8)


def grainy(w, h, n=4, amp=40):
    """Strong noise over a drifting texture: inter blocks with all 16 coefficients coded."""
    base = drift(w, h, [(1, 0)] * (n - 1), seed=8).astype(np.int64)
    rng = np.random.default_rng(9)
    return (base + rng.integers(-amp, amp + 1, base.shape)).clip(0, 255).astype(np.uint8)


def avatar_motion(w, h, n=3):
    return np.stack([shifted(hc.avatar_like(w, h), k, k // 2) for k in range(n)])


def sequences(large: bool = True):
    """[(name, frames (K, H, W, 3) uint8, qp, gop)]."""
    items = [("static64x48", static(64, 48, 4), 20, 4),
             ("flat64x48", np.stack([hc.flat(64, 48)] * 3), 20, 3),
             ("drift64x48", drift(64, 48, [(1, 0), (0, 2), (-3, 1), (2, -2)]), 14, 8),
             ("pan80x64", pan(80, 64), 20, 16),
             ("scene_cut48x32", scene_cut(48, 32), 26, 5),
             ("noise48x32", noisy(48, 32), 0, 3),
             ("noise48x32@30", noisy(48, 32), 30, 3),
             ("soft64x32", soft(64, 32, 5), 24, 5),
             ("soft64x32@40", soft(64, 32, 5), 40, 2),
             ("grainy64x32", grainy(64, 32), 8, 4),
             ("cut_to_escapes64x32", np.stack([hc.gradient(64, 32), hc.dc_escapes()]), 0, 2),
             ("wrap16x16", drift(16, 16, [(1, 1)] * 19), 20, 20),
             ("odd18x34", drift(18, 34, [(1, 0), (0, 1), (-1, 1)]), 18, 3)]
    if large:
        items += [("avatar550x802", avatar_motion(550, 802), 20, 25)]
    return items
