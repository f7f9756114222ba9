"""CPU: the tile-packed lossless frame format (oracle/frame_codec.py, the numpy restatement csrc/frames.cu is held to).

One tiny frame's record is pinned byte by byte below: it documents the format.  Round trips are bit-exact on the
frames that stress each part of it (every width 8, constant tiles, mod-256 wrap, a lone spike, binary masks) at
ragged and full sizes; edge replication adds no residual; record sizes follow 8 + 32 sum(b), and no frame exceeds
n_tiles * 1036 + 8 bytes with its index."""
import numpy as np
import pytest

from oracle import frame_codec as fc

SIZES = [(1, 1), (1, 17), (17, 1), (15, 16), (550, 802), (1080, 1920)]


def _frames(kind, F, H, W, seed=0):
    """(gt (F,3,H,W), mask (F,1,H,W)) uint8 of one kind."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (F, 3, H, W), dtype=np.uint8), rng.integers(0, 256, (F, 1, H, W), dtype=np.uint8)
    if kind == "constant":
        c = rng.integers(0, 256, (F, 4, 1, 1), dtype=np.uint8)
        v = np.broadcast_to(c, (F, 4, H, W)).copy()
        return v[:, :3], v[:, 3:]
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    if kind == "ramp":   # steps that wrap past 255 inside tiles, a different slope per plane
        v = np.stack([(xx * (5 + 3 * p) + yy * (11 + 2 * p) + 40 * p) % 256 for p in range(4)]).astype(np.uint8)
        return np.broadcast_to(v[:3], (F, 3, H, W)).copy(), np.broadcast_to(v[3:], (F, 1, H, W)).copy()
    if kind == "spike":   # one flat tile value with one pixel 255 - value, per plane
        v = np.full((F, 4, H, W), 7, np.uint8)
        v[:, :, H // 2, W // 2] = 248
        return v[:, :3], v[:, 3:]
    if kind == "binary":   # an ellipse mask of 0 / 255 and the background where it is 0
        inside = ((xx - W / 2) / max(W * 0.35, 1)) ** 2 + ((yy - H / 2) / max(H * 0.4, 1)) ** 2 < 1
        m = np.where(inside, 255, 0).astype(np.uint8)
        gt = rng.integers(0, 256, (F, 3, H, W), dtype=np.uint8)
        gt[:, :, ~inside] = 255
        return gt, np.broadcast_to(m, (F, 1, H, W)).copy()
    raise ValueError(kind)


def test_pinned_record_of_a_tiny_frame():
    """A 2x3 frame: R = [[10, 12, 11], [10, 10, 10]], G = 0, B = 200, no mask (M = 255).
    R: base 10; the edge-replicated q has row 0 = 0 2 1 1 1 ..., every other row 0; the nonzero differences are
    d(0,1) = 2, d(0,2) = -1, d(1,1) = -2, d(1,2) = 1 -> zigzag 4, 1, 3, 2 -> width 3.  Value i sits at bits [3i, 3i+3):
    i=1 -> bit 5, i=2 -> bit 6 (byte 0 = 0x60); i=17 (3) -> bits 51, 52, i=18 (2) -> bit 55 (byte 6 = 0x98).
    G, B, M are constant: width 0, no payload."""
    gt = np.zeros((3, 2, 3), np.uint8)
    gt[0] = [[10, 12, 11], [10, 10, 10]]
    gt[2] = 200
    rec, off = fc.encode_frame(fc.planes_of(gt))
    want = np.zeros(8 + 96, np.uint8)
    want[:8] = [10, 0, 200, 255, 0x03, 0x00, 0, 0]
    want[8 + 0], want[8 + 6] = 0x60, 0x98
    assert off.tolist() == [0]
    assert rec.tolist() == want.tolist()
    assert np.array_equal(fc.decode_frame(rec, off, 2, 3), fc.planes_of(gt))


@pytest.mark.parametrize("kind", ["noise", "constant", "ramp", "spike", "binary"])
@pytest.mark.parametrize("H,W", SIZES)
def test_round_trip_is_bit_exact(kind, H, W):
    F = 2 if H * W <= 550 * 802 else 1
    gt, mask = _frames(kind, F, H, W, seed=H + W)
    arena, base, off = fc.encode_frames(gt, mask)
    ids = [F - 1, 0, F - 1] if F > 1 else [0, 0]
    g2, m2 = fc.decode_frames(arena, base, off, ids, H, W)
    assert np.array_equal(g2, gt[ids]) and np.array_equal(m2, mask[ids])
    T = int(np.prod(fc.tiles_of(H, W)))
    assert off.shape == (F, T) and base[0] == 0 and arena.size % 8 == 0
    widths = fc.transform(fc._tiles(fc.planes_of(gt[0], mask[0])))[2]
    if kind == "noise" and H >= 16 and W >= 16:   # a whole tile of noise: every plane at width 8
        assert (widths[0] == 8).all()
    if kind == "constant":   # 8-byte records: bases and widths only
        assert (widths == 0).all() and arena.size == F * T * 8
    if kind == "spike":
        assert int((widths > 0).sum()) <= 4 * 4   # the spike's tile (and its neighbours' edges) only


def test_mask_none_is_255():
    gt, _ = _frames("noise", 1, 20, 33)
    arena, base, off = fc.encode_frames(gt, None)
    g2, m2 = fc.decode_frames(arena, base, off, [0], 20, 33)
    assert np.array_equal(g2, gt) and (m2 == 255).all()


@pytest.mark.parametrize("H,W", [(17, 1), (1, 17), (15, 16), (21, 35), (550, 802)])
def test_edge_replication_adds_no_residual(H, W):
    """Past the frame's edge every residual is zero, so a ragged tile is as wide as its in-frame pixels need."""
    gt, mask = _frames("noise", 1, H, W, seed=3)
    planes = fc.planes_of(gt[0], mask[0])
    ty, tx = fc.tiles_of(H, W)
    _, z, widths = fc.transform(fc._tiles(planes))
    z = z.reshape(ty, tx, 4, 16, 16).transpose(2, 0, 3, 1, 4).reshape(4, ty * 16, tx * 16)
    assert not z[:, H:, :].any() and not z[:, :, W:].any()
    inner = z[:, :H, :W]
    zt = np.zeros((4, ty * 16, tx * 16), np.uint8)
    zt[:, :H, :W] = inner
    zt = zt.reshape(4, ty, 16, tx, 16).transpose(1, 3, 0, 2, 4).reshape(ty * tx, 4, 256)
    assert np.array_equal(widths, fc._BITLEN[zt.max(axis=-1)])
    # zero padding instead of replication would code the step down to 0 at the edge
    pad = np.pad(planes, ((0, 0), (0, ty * 16 - H), (0, tx * 16 - W)))
    if (ty * 16 - H) or (tx * 16 - W):
        zpad = fc.transform(pad.reshape(4, ty, 16, tx, 16).transpose(1, 3, 0, 2, 4).reshape(ty * tx, 4, 16, 16))[1]
        assert zpad.reshape(ty, tx, 4, 16, 16).transpose(2, 0, 3, 1, 4).reshape(4, ty * 16, tx * 16)[:, H:, :].any() \
            or zpad.reshape(ty, tx, 4, 16, 16).transpose(2, 0, 3, 1, 4).reshape(4, ty * 16, tx * 16)[:, :, W:].any()


@pytest.mark.parametrize("kind", ["noise", "constant", "ramp", "spike", "binary"])
def test_record_sizes_and_the_frame_bound(kind):
    H, W = 47, 70
    gt, mask = _frames(kind, 1, H, W, seed=9)
    rec, off = fc.encode_frame(fc.planes_of(gt[0], mask[0]))
    widths = fc.transform(fc._tiles(fc.planes_of(gt[0], mask[0])))[2]
    T = widths.shape[0]
    sizes = [fc.record_bytes(w) for w in widths]
    assert all(s == 8 + 32 * int(w.sum()) and s % 8 == 0 and s <= fc.RECORD_MAX for s, w in zip(sizes, widths))
    assert off.tolist() == (np.cumsum([0] + sizes[:-1]) // 8).tolist() and rec.size == sum(sizes)
    assert rec.size + 4 * T + 8 <= fc.frame_bound(T)
    if kind == "noise":   # interior tiles at width 8 everywhere
        assert max(sizes) == fc.RECORD_MAX


def test_worst_case_meets_the_bound_exactly():
    gt, mask = _frames("noise", 1, 64, 64, seed=1)
    rec, off = fc.encode_frame(fc.planes_of(gt[0], mask[0]))
    T = 16
    assert rec.size == T * fc.RECORD_MAX and rec.size + 4 * T + 8 == fc.frame_bound(T) == T * 1036 + 8
