"""Images and sizes for the H.264 encoder's tests, built to reach every path oracle/h264.py reports: each coeff_token
table, level_prefix 0..15 at every suffixLength, every total_zeros and run_before table, every luma and chroma mode,
I_PCM and emulation-prevention bytes.

    for name, rgb, qp in corpus(): ...      # (H, W, 3) uint8 numpy images and their QP

Limited-range black is Y = 16, so I_PCM samples are never zero bytes; the emulation-prevention image instead holds
flat 4x4 blocks whose only coefficients are large luma DC levels: their 12-bit level escapes with zero suffixes put
runs of more than 22 zero bits into the slice.
"""
from __future__ import annotations

import numpy as np

QPS = (0, 10, 20, 30, 40, 51)
SMALL_SIZES = ((2, 2), (16, 16), (18, 34), (32, 2), (2, 32))
LARGE_SIZES = ((550, 802), (1920, 1080))


def flat(w, h, rgb=(90, 160, 220)):
    return np.broadcast_to(np.array(rgb, np.uint8), (h, w, 3)).copy()


def gradient(w, h):
    """Smooth ramps: Plane prediction wins away from the edges."""
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y) * 127 // max(w + h - 2, 1))],
                    -1).astype(np.uint8)


def stripes(w, h, vertical: bool):
    """Columns (V wins) or rows (H wins) of pseudo-random colours."""
    rng = np.random.default_rng(3 if vertical else 4)
    n = w if vertical else h
    line = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    return np.broadcast_to(line[None] if vertical else line[:, None], (h, w, 3)).copy()


def noise(w, h, seed=0, amp=255):
    rng = np.random.default_rng(seed)
    base = 128 - amp // 2
    return (base + rng.integers(0, amp + 1, (h, w, 3))).clip(0, 255).astype(np.uint8)


def textured(w, h, seed=1):
    """Low-amplitude texture over a gradient: many small levels, every total_zeros and run_before table."""
    rng = np.random.default_rng(seed)
    g = gradient(w, h).astype(np.int64)
    return (g + rng.integers(-12, 13, (h, w, 3)) * (rng.random((h, w, 1)) < 0.3)).clip(0, 255).astype(np.uint8)


def dc_escapes(w=64, h=32, seed=5):
    """Flat 4x4 blocks of extreme grey levels: only luma DC levels, large enough for 12-bit escapes."""
    rng = np.random.default_rng(seed)
    v = rng.choice(np.array([0, 255], np.uint8), (h // 4, w // 4))
    return np.repeat(np.repeat(v, 4, 0), 4, 1)[..., None].repeat(3, -1)


def avatar_like(w, h, seed=2):
    """A smooth head-sized blob with shading over a white background, the look of a render."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    cx, cy, r = w / 2, h / 2.2, min(w, h) / 3
    d = np.sqrt(((x - cx) / r) ** 2 + ((y - cy) / (1.3 * r)) ** 2)
    shade = np.clip(1.1 - d, 0, 1)
    skin = np.stack([200 * shade + 40, 150 * shade + 30, 120 * shade + 25], -1)
    rng = np.random.default_rng(seed)
    skin += rng.normal(0, 3, skin.shape)
    return np.where((d < 1)[..., None], skin, 255).clip(0, 255).astype(np.uint8)


def small_images():
    out = []
    for w, h in SMALL_SIZES:
        out += [(f"flat{w}x{h}", flat(w, h)), (f"gradient{w}x{h}", gradient(w, h)),
                (f"noise{w}x{h}", noise(w, h, seed=w * 7 + h))]
    out += [("vstripes48x32", stripes(48, 32, True)), ("hstripes48x32", stripes(48, 32, False)),
            ("gradient64x48", gradient(64, 48)), ("textured64x64", textured(64, 64)),
            ("noise48x48", noise(48, 48, seed=9)), ("softnoise64x32", noise(64, 32, seed=11, amp=24)),
            ("dc_escapes64x32", dc_escapes())]
    return out


def corpus(large: bool = True):
    """[(name, rgb (H,W,3) uint8, qp)]: every small image at every QP, and the large sizes at a few."""
    items = [(f"{n}@{qp}", img, qp) for n, img in small_images() for qp in QPS]
    if large:
        items += [("avatar550x802@20", avatar_like(550, 802), 20), ("textured1920x1080@30", textured(1920, 1080), 30)]
    return items
