"""Frame sequences for the I_NxN H.264 stream (tests/h264_intra4x4_oracle.py, gab200_h264_encode_flags with
GAB200_H264_INTRA4X4): the deblocked corpus (tests/h264_deblock_corpus.py), which brings I_16x16, I_PCM, P_L0_16x16
and P_Skip neighbours, plus fine directional texture that every Intra_4x4 mode predicts best somewhere, on the
picture's top row and left and right columns, and a detailed avatar.

    for name, frames, qp, gop in sequences(): ...      # frames (K, H, W, 3) uint8
"""
from __future__ import annotations

import numpy as np

from tests import h264_corpus as hc
from tests import h264_deblock_corpus as dc
from tests import h264_inter_corpus as ic


def directions(w, h, seed=3):
    """Tiles of sharp stripes at eight angles with random phase and period, so that each 4x4 block has one
    direction the modes can follow."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w, 3), np.uint8)
    for ty in range(0, h, 8):
        for tx in range(0, w, 8):
            a = rng.uniform(0, np.pi)
            period = rng.uniform(3, 9)
            v = np.cos(a) * xx[ty:ty + 8, tx:tx + 8] + np.sin(a) * yy[ty:ty + 8, tx:tx + 8]
            lum = np.where(np.sin(2 * np.pi * v / period + rng.uniform(0, 6)) > 0, 220, 30)
            img[ty:ty + 8, tx:tx + 8] = np.stack([lum, (lum + rng.integers(0, 60)) % 256, 255 - lum], -1)
    return img


def moving_directions(w, h, n=3):
    f = [directions(w, h)]
    for dx, dy in [(1, 0), (0, 2), (3, 1)][:n - 1]:
        f.append(ic.shifted(f[-1], dx, dy))
    f[-1] = f[-1].copy()
    f[-1][h // 3:h // 3 + 16, w // 3:w // 3 + 16] = directions(16, 16, seed=9)   # an uncovered region in a P picture
    return np.stack(f)


def lower_halves(w, h):
    """Flat upper halves and striped lower halves of every macroblock: coded_block_pattern with only the lower 8x8
    quadrants."""
    img = directions(w, h, seed=5)
    img[(np.arange(h) % 16) < 8] = (90, 160, 220)
    return img


def sequences(large: bool = True):
    """[(name, frames (K, H, W, 3) uint8, qp, gop)]."""
    items = dc.sequences(large=False)
    items += [("directions64x48", np.stack([directions(64, 48)]), 20, 1),
              ("directions_motion80x64", moving_directions(80, 64), 26, 3),
              ("lower_halves48x32", np.stack([lower_halves(48, 32)]), 20, 1),
              ("textured_lowqp48x32", np.stack([hc.textured(48, 32, seed=4)] * 2), 4, 2),
              ("avatar_detail96x64", ic.avatar_motion(96, 64, 3), 20, 3)]
    if large:
        items += [("avatar550x802", ic.avatar_motion(550, 802), 26, 25)]
    return items
