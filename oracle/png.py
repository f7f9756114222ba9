"""numpy restatement of the PNG encoder's decisions (gaussianavatars_b200/csrc/png.cu): the row filters, the rule that
picks one per row, the segmentation of the filtered stream and the worst-case file size.

The rule is libpng's minimum-sum-of-absolute-values heuristic: each filtered byte v counts v < 128 ? v : 256 - v, the
row takes the filter with the least sum, and a tie goes to the lowest filter id (0 None, 1 Sub, 2 Up, 3 Average,
4 Paeth).  PIL does not follow this rule exactly, so its files are not the oracle.
"""
from __future__ import annotations

import numpy as np

BPP = 3                  # bytes per pixel: 8-bit RGB
SEGMENT = 32768          # filtered bytes per deflate block
FILTERS = ("none", "sub", "up", "average", "paeth")


def filter_row(cur: np.ndarray, prev: np.ndarray | None, ftype: int) -> np.ndarray:
    """Row `cur` (3W uint8) filtered with filter `ftype` against the row above (None: the first row, all zero)."""
    x = cur.astype(np.int32)
    b = np.zeros_like(x) if prev is None else prev.astype(np.int32)
    a = np.concatenate([np.zeros(BPP, np.int32), x[:-BPP]])[:x.size]
    c = np.concatenate([np.zeros(BPP, np.int32), b[:-BPP]])[:x.size]
    if ftype == 0:
        pred = np.zeros_like(x)
    elif ftype == 1:
        pred = a
    elif ftype == 2:
        pred = b
    elif ftype == 3:
        pred = (a + b) >> 1
    elif ftype == 4:
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    else:
        raise ValueError(f"a PNG filter id is 0..4, got {ftype}")
    return ((x - pred) & 255).astype(np.uint8)


def row_cost(filtered: np.ndarray) -> int:
    """The heuristic's sum: every byte read as a signed magnitude."""
    v = filtered.astype(np.int64)
    return int(np.where(v < 128, v, 256 - v).sum())


def choose_filter(cur: np.ndarray, prev: np.ndarray | None) -> tuple:
    """(filter id, filtered row) the rule picks for one row."""
    best, best_row, best_cost = 0, None, None
    for f in range(5):
        row = filter_row(cur, prev, f)
        cost = row_cost(row)
        if best_cost is None or cost < best_cost:
            best, best_row, best_cost = f, row, cost
    return best, best_row


def filter_image(rgb: np.ndarray) -> tuple:
    """(filter ids (H,), filtered stream (H * (3W + 1),) uint8) of an (H, W, 3) uint8 image."""
    H, W, _ = rgb.shape
    rows = rgb.reshape(H, 3 * W)
    ids, out = np.zeros(H, np.uint8), np.zeros((H, 3 * W + 1), np.uint8)
    for y in range(H):
        f, row = choose_filter(rows[y], rows[y - 1] if y else None)
        ids[y], out[y, 0], out[y, 1:] = f, f, row
    return ids, out.reshape(-1)


def filtered_bytes(width: int, height: int) -> int:
    return height * (3 * width + 1)


def segments(width: int, height: int) -> int:
    """Deflate blocks of a file: one per SEGMENT filtered bytes, the last one shorter."""
    return -(-filtered_bytes(width, height) // SEGMENT)


def png_bound(width: int, height: int) -> int:
    """The largest file of a width x height image: signature 8, IHDR 25, IDAT chunk 12, zlib header 2 and Adler-32 4,
    IEND 12, and the deflate stream, at most every block stored (3 header bits, <= 7 bits of padding, LEN and NLEN:
    42 bits <= 6 bytes per block) -- 63 + n + 6 S."""
    if width <= 0 or height <= 0:
        raise ValueError(f"a PNG has a positive size, got {width}x{height}")
    n = filtered_bytes(width, height)
    return 63 + n + 6 * segments(width, height)
