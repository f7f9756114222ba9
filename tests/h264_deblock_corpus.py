"""Frame sequences for the deblocked H.264 stream (tests/h264_deblock_oracle.py, gab200_h264_encode_deblocked): the P
corpus (tests/h264_inter_corpus.py), which reaches every bS, both filters and their clipping, plus I_PCM macroblocks
beside I_16x16 ones and a soft avatar at a high QP.

    for name, frames, qp, gop in sequences(): ...      # frames (K, H, W, 3) uint8
"""
from __future__ import annotations

import numpy as np

from tests import h264_corpus as hc
from tests import h264_inter_corpus as ic

# the QPs FFmpeg referees the filter at: alpha' is 0 below 16, and 51 is the top of the tables
QPS = (0, 15, 16, 20, 26, 32, 38, 45, 51)


def pcm_beside_intra(w=64, h=32):
    """Noise on the left (I_PCM at low QPs), a gradient on the right: edges with an I_PCM side."""
    a = hc.noise(w, h, seed=5)
    a[:, w // 2:] = hc.gradient(w - w // 2, h)
    return np.stack([a, ic.shifted(a, 1, 0)])


def sequences(large: bool = True):
    """[(name, frames (K, H, W, 3) uint8, qp, gop)]."""
    items = ic.sequences(large=False)
    items += [("pcm_beside_intra64x32", pcm_beside_intra(), 8, 2),
              ("avatar96x64@32", ic.avatar_motion(96, 64, 4), 32, 4)]
    if large:
        items += [("avatar550x802", ic.avatar_motion(550, 802), 26, 25)]
    return items
