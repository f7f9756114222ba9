"""numpy restatement of the tile-packed lossless frame codec of gaussianavatars_b200.frames (csrc/frames.cu).
TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product.

A frame is four uint8 planes: R, G, B of the composited ground truth (planar) and M, the alpha bytes (255 for a frame
stored without a mask).  Each plane is cut into 16x16 tiles in row-major tile order; a tile's values replicate the
frame's last row / column past its edge:

    v(y, x) = P(min(16 ty + y, H - 1), min(16 tx + x, W - 1))

and are coded, mod 256, as

    base = v(0, 0),  q = v - base,  d(y, x) = q(y, x) - q(y, x-1) - q(y-1, x) + q(y-1, x-1)   (q = 0 off the tile)
    z = zigzag((int8) d) = ((s << 1) ^ (s >> 7)) & 0xff,  b = bit length of max z over the tile's 256 values

The inverse is a 2-D inclusive prefix sum of d (mod 256) plus the base.

Tile record (8-byte aligned): bytes 0-3 the four bases; bytes 4-5 a little-endian uint16 holding the four widths,
plane p in bits 4p..4p+3; bytes 6-7 zero; then the R, G, B and M payloads, 32 b bytes each, value i = 16 y + x at bits
[i b, i b + b) of a little-endian bit stream (bit j is bit j % 8 of byte j / 8).  A record is 8 + 32 sum(b) bytes.

Index: `frame_base` (int64 per frame, a byte offset into the arena) and `tile_off` (uint32 per (frame, tile), in 8-byte
units from the frame's base).  A frame costs at most n_tiles * 1036 + 8 bytes, records and index included.
"""
import numpy as np

TILE = 16
PLANES = 4
RECORD_MAX = 8 + 32 * 8 * PLANES          # 1032 bytes for the 1024 values of a tile
_BITLEN = np.array([int(v).bit_length() for v in range(256)], dtype=np.int64)


def tiles_of(height: int, width: int):
    return (height + TILE - 1) // TILE, (width + TILE - 1) // TILE


def frame_bound(n_tiles: int) -> int:
    """The most bytes one frame can take: every record at 1032 bytes, its 4-byte offset, and the 8-byte frame base."""
    return n_tiles * (RECORD_MAX + 4) + 8


def record_bytes(widths) -> int:
    return 8 + 32 * int(np.sum(widths))


def planes_of(gt: np.ndarray, mask=None) -> np.ndarray:
    """(3,H,W) ground truth and (1,H,W) alpha (None: 255) -> the (4,H,W) uint8 planes a frame stores."""
    gt = np.asarray(gt, dtype=np.uint8)
    m = np.full((1,) + gt.shape[1:], 255, np.uint8) if mask is None else np.asarray(mask, np.uint8).reshape(1, *gt.shape[1:])
    return np.concatenate([gt, m], axis=0)


def _tiles(planes: np.ndarray) -> np.ndarray:
    """(4,H,W) -> (T,4,16,16), edge-replicated, row-major tile order."""
    _, H, W = planes.shape
    ty, tx = tiles_of(H, W)
    v = np.pad(planes, ((0, 0), (0, ty * TILE - H), (0, tx * TILE - W)), mode="edge")
    return v.reshape(PLANES, ty, TILE, tx, TILE).transpose(1, 3, 0, 2, 4).reshape(ty * tx, PLANES, TILE, TILE)


def transform(v: np.ndarray):
    """(T,4,16,16) tile values -> bases (T,4), zigzag residuals z (T,4,16,16) and widths (T,4)."""
    base = v[..., 0, 0]
    q = (v - base[..., None, None]).astype(np.uint8)
    left = np.zeros_like(q)
    left[..., :, 1:] = q[..., :, :-1]
    up = np.zeros_like(q)
    up[..., 1:, :] = q[..., :-1, :]
    diag = np.zeros_like(q)
    diag[..., 1:, 1:] = q[..., :-1, :-1]
    d = (q - left - up + diag).astype(np.uint8)                      # mod 256
    s = d.view(np.int8).astype(np.int32)
    z = (((s << 1) ^ (s >> 7)) & 0xFF).astype(np.uint8)
    widths = _BITLEN[z.reshape(z.shape[0], PLANES, -1).max(axis=-1)]
    return base, z, widths


def inverse(base: np.ndarray, z: np.ndarray) -> np.ndarray:
    """bases (T,4) and residuals (T,4,16,16) -> the tile values."""
    zi = z.astype(np.int32)
    d = ((zi >> 1) ^ -(zi & 1)) & 0xFF
    q = np.cumsum(np.cumsum(d, axis=-1), axis=-2)
    return ((q + base[..., None, None].astype(np.int32)) & 0xFF).astype(np.uint8)


def _pack(z: np.ndarray, b: int) -> np.ndarray:
    """(n,256) values of width b -> (n, 32 b) bytes of the little-endian bit stream."""
    bits = (z[..., None].astype(np.uint32) >> np.arange(b, dtype=np.uint32)) & 1
    return np.packbits(bits.reshape(z.shape[0], -1).astype(np.uint8), axis=-1, bitorder="little")


def _unpack(raw: np.ndarray, b: int) -> np.ndarray:
    bits = np.unpackbits(raw, axis=-1, bitorder="little").reshape(raw.shape[0], 256, b).astype(np.uint32)
    return (bits << np.arange(b, dtype=np.uint32)).sum(axis=-1).astype(np.uint8)


def encode_frame(planes: np.ndarray):
    """(4,H,W) uint8 planes -> (records: uint8 bytes of the frame's records, tile_off: (n_tiles,) uint32 in 8-byte
    units from the frame's first byte)."""
    base, z, widths = transform(_tiles(planes))
    T = base.shape[0]
    zf = z.reshape(T, PLANES, 256)
    payload = {}
    for b in range(1, 9):
        sel = np.argwhere(widths == b)
        if len(sel):
            packed = _pack(zf[sel[:, 0], sel[:, 1]], b)
            for (t, p), row in zip(map(tuple, sel), packed):
                payload[(t, p)] = row
    out, offs, pos = [], np.zeros(T, np.uint32), 0
    for t in range(T):
        hdr = np.zeros(8, np.uint8)
        hdr[:4] = base[t]
        w = int(sum(int(widths[t, p]) << (4 * p) for p in range(PLANES)))
        hdr[4], hdr[5] = w & 0xFF, w >> 8
        rec = [hdr] + [payload[(t, p)] for p in range(PLANES) if widths[t, p] > 0]
        offs[t] = pos // 8
        out.extend(rec)
        pos += record_bytes(widths[t])
    return np.concatenate(out), offs


def decode_frame(records: np.ndarray, tile_off: np.ndarray, height: int, width: int) -> np.ndarray:
    """The inverse of encode_frame: the (4,H,W) planes of one frame's records."""
    records = np.asarray(records, np.uint8)
    start = np.asarray(tile_off, np.int64) * 8
    T = start.shape[0]
    hdr = records[start[:, None] + np.arange(8)]
    base = hdr[:, :4]
    w16 = hdr[:, 4].astype(np.int64) | (hdr[:, 5].astype(np.int64) << 8)
    widths = np.stack([(w16 >> (4 * p)) & 0xF for p in range(PLANES)], axis=1)
    pstart = start[:, None] + 8 + 32 * (np.cumsum(widths, axis=1) - widths)
    z = np.zeros((T, PLANES, 256), np.uint8)
    for b in range(1, 9):
        t, p = np.nonzero(widths == b)
        if len(t):
            z[t, p] = _unpack(records[pstart[t, p][:, None] + np.arange(32 * b)], b)
    v = inverse(base, z.reshape(T, PLANES, TILE, TILE))
    ty, tx = tiles_of(height, width)
    full = v.reshape(ty, tx, PLANES, TILE, TILE).transpose(2, 0, 3, 1, 4).reshape(PLANES, ty * TILE, tx * TILE)
    return np.ascontiguousarray(full[:, :height, :width])


def encode_frames(gt: np.ndarray, mask=None):
    """(F,3,H,W) ground truth and (F,1,H,W) alpha (None: 255) -> (arena uint8, frame_base (F,) int64 byte offsets,
    tile_off (F, n_tiles) uint32): the frames' records back to back from byte 0, in frame order."""
    gt = np.asarray(gt, np.uint8)
    parts, bases, offs, pos = [], [], [], 0
    for f in range(gt.shape[0]):
        rec, off = encode_frame(planes_of(gt[f], None if mask is None else mask[f]))
        parts.append(rec)
        bases.append(pos)
        offs.append(off)
        pos += rec.size
    return np.concatenate(parts), np.array(bases, np.int64), np.stack(offs)


def decode_frames(arena, frame_base, tile_off, ids, height: int, width: int):
    """(gt (K,3,H,W), mask (K,1,H,W)) of frames `ids` of an arena and its index."""
    arena = np.asarray(arena, np.uint8)
    out = np.stack([decode_frame(arena[int(frame_base[i]):], tile_off[i], height, width) for i in ids])
    return np.ascontiguousarray(out[:, :3]), np.ascontiguousarray(out[:, 3:])
