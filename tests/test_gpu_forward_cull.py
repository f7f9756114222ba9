"""-m gpu: the forward blend's box cull (blend.cu `reaches_rect` on SplatRec q2.yz) and its block masks, checked
against the records and the sorted lists the forward really used, separately from the blend's outputs.  Skipping, per
warp, the splats whose box misses the warp's pixels changes no output bit exactly when the box test below has zero
misses.

Per frame the test reads back the SplatRec of every splat, the sorted instance list, the per-instance block masks,
final_T and n_contrib, and evaluates in float32 numpy, for every instance and every pixel of its tile, the walk's
exponent `pw = fmaf(C' dy, dy, fmaf(B', dy, A' dx) dx)` and alpha.  ex2.approx and the rounding of pw are replaced by
bounds (`_pixel_bounds`), which give a "possibly live" and a "certainly live" set per (instance, pixel).  Asserted:
  * every (instance, 8x4 block) with a possibly-live pixel passes the box test: the cull never drops a splat the
    unculled walk would have blended (zero misses);
  * the block masks the forward wrote lie between the blocks whose pixels certainly and possibly took the instance
    before their n_contrib, and inside the box-live blocks;
  * no pixel's n_contrib points at an entry that is box-dead for the pixel's block.
Frames: the adversarial scenes (degenerate conics, opacity at 1/255, centres on block edges, huge and sub-pixel
splats, saturating stacks, ragged sizes), each also through the narrowed, dollied and mirrored cameras of
tests/bound_rigs.py, and the headline 100k-splat 1080p frame, for which the fraction of each warp's walk that the box
test skips is printed (run with -s)."""
import math

import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import bound_rigs as BR
from tests import helpers as h

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
ALPHA_MIN = float(F32(1.0) / F32(255.0))
LOG2E = F32(1.4426950408889634)


def _read_frame(P, W, H):
    """The last forward's records, sorted ids, ranges, block masks, final_T and n_contrib (needs a training forward:
    keep_last_state(True) and inputs that require grad)."""
    from gaussianavatars_b200 import rasterizer as R

    _, vals, ranges, n = R.export_last_binning()
    a, st, holder, _ = R._last
    assert holder is not None, "the frame was not a training forward"
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tiles = gx * gy
    geom = h.buffer(holder, st.geom_buffer)
    rec = geom[: P * 48].view(torch.float32).reshape(P, 12).cpu().numpy()
    nb = max(int(st.binning_capacity), 1) + 320
    off = h.carve([4 * nb] * 4 + [nb])[4]
    strip = h.buffer(holder, st.binning_buffer)[off: off + n].cpu().numpy()
    offs = h.carve([(tiles + 1) * 8, tiles * 4, 16, tiles * 4, tiles * 4, W * H * 4, W * H * 4])
    img = h.buffer(holder, st.image_buffer)
    final_T = img[offs[5]: offs[5] + 4 * W * H].view(torch.float32).reshape(H, W).cpu().numpy()
    n_contrib = img[offs[6]: offs[6] + 4 * W * H].view(torch.int32).reshape(H, W).cpu().numpy()
    return dict(rec=rec, vals=vals.cpu().numpy().view(np.uint32), ranges=ranges.cpu().numpy().view(np.uint32),
                strip=strip, final_T=final_T, n_contrib=n_contrib, W=W, H=H, n=n)


def _fma32(a, b, c):
    """float32 fmaf through float64: the product of two floats is exact there, the sum is rounded twice (the error
    bound in `_pixel_bounds` covers the second rounding)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def _pixel_bounds(r, fx, fy):
    """(possibly, certainly) live per (instance, pixel): r (M,12) records, fx / fy (256,) pixel centres of the tile
    (M,256).  The walk's test is pw <= 0 and min(0.99, op * ex2.approx(pw)) >= 1/255; pw's rounding is bounded by
    2^-21 of the sum of its terms' magnitudes, ex2.approx's relative error and the product's rounding by 2^-20."""
    px, py, Ap, Bp, Cp, op = (r[:, k:k + 1] for k in (0, 1, 2, 3, 4, 5))
    with np.errstate(all="ignore"):   # huge and degenerate records overflow to inf / nan, as they do on the device
        dx = px - fx
        dy = py - fy
        tA = Ap * dx
        pw = _fma32(Cp * dy, dy, _fma32(Bp, dy, tA) * dx).astype(np.float64)
        e = 2.0 ** -21 * (np.abs(tA.astype(np.float64) * dx) + np.abs(Bp.astype(np.float64) * dx * dy)
                          + np.abs(Cp.astype(np.float64) * dy * dy))
        op64 = op.astype(np.float64)
        hi = np.minimum(0.99, op64 * np.exp2(pw + e) * (1 + 2.0 ** -20))
        lo = np.minimum(0.99, op64 * np.exp2(pw - e) * (1 - 2.0 ** -20))
        possibly = (pw - e <= 0) & (hi >= ALPHA_MIN)
        certainly = (pw + e <= 0) & (lo >= ALPHA_MIN)
    return possibly, certainly


def _box(r, x0, x1, y0, y1):
    """The box test in float32 (distance from the centre to the rectangle, per axis, against rx / ry; -1 never
    passes, NaN always does): (M,1) records against (8,) block rectangles -> (M,8)."""
    px, py, rx, ry = (r[:, k:k + 1] for k in (0, 1, 9, 10))
    ex = np.fmax(np.fmax(x0 - px, px - x1), F32(0))
    ey = np.fmax(np.fmax(y0 - py, py - y1), F32(0))
    return ~(ex > rx) & ~(ey > ry)


# pixel (ly, lx) of a tile, row-major; its block bit 2 * band + half (BandGeom::bit)
_LY, _LX = np.divmod(np.arange(256), 16)
_BIT = 2 * (_LY // 4) + _LX // 8
_BLK_ONEHOT = (_BIT[:, None] == np.arange(8)[None, :])          # (256, 8)
_B_HALF, _B_BAND = np.arange(8) % 2, np.arange(8) // 2


def _blocks(pix):
    """(M,256) per-pixel -> (M,8) any over each block's 32 pixels."""
    return (pix.astype(np.uint8) @ _BLK_ONEHOT.astype(np.uint8)) > 0


def analyse(fr, what, chunk=8192):
    """Runs every check on one frame; returns the walk counts (entries inside each 8x4 block's walk, and how many of
    them the box test and a per-pixel exact test would skip)."""
    rec, vals, ranges, strip = fr["rec"], fr["vals"], fr["ranges"], fr["strip"]
    W, H, n = fr["W"], fr["H"], fr["n"]
    nc = fr["n_contrib"].astype(np.int64)
    gx = (W + 15) // 16
    lens = (ranges[:, 1].astype(np.int64) - ranges[:, 0])
    tile_of = np.repeat(np.arange(len(ranges)), lens)
    assert tile_of.size == n
    pos = np.arange(n, dtype=np.int64) - ranges[tile_of, 0].astype(np.int64)
    # per tile pixel: global index (or -1 outside the image) and n_contrib (0 outside)
    tx, ty = np.arange(len(ranges)) % gx, np.arange(len(ranges)) // gx
    X = tx[:, None] * 16 + _LX[None, :]
    Y = ty[:, None] * 16 + _LY[None, :]
    inside = (X < W) & (Y < H)
    nc_tile = np.where(inside, nc[np.minimum(Y, H - 1), np.minimum(X, W - 1)], 0)      # (tiles, 256)
    nc_max = nc_tile.max(axis=1)
    box_all = np.zeros((n, 8), bool)
    poss_all = np.zeros((n, 8), bool)
    sat = np.where(inside, lens[:, None], -1)      # first possibly-live entry at or past n_contrib: where the pixel stops
    for s in range(0, n, chunk):
        sl = slice(s, min(n, s + chunk))
        t, p = tile_of[sl], pos[sl]
        r = rec[vals[sl]]
        fx = X[t].astype(F32)
        fy = Y[t].astype(F32)
        possibly, certainly = _pixel_bounds(r, fx, fy)
        possibly &= inside[t]
        certainly &= inside[t]
        x0 = (tx[t, None] * 16 + 8 * _B_HALF[None, :]).astype(F32)
        y0 = (ty[t, None] * 16 + 4 * _B_BAND[None, :]).astype(F32)
        box = _box(r, x0, x0 + F32(7), y0, y0 + F32(3))
        poss_b = _blocks(possibly)
        miss = poss_b & ~box
        if miss.any():
            i, b = np.argwhere(miss)[0]
            raise AssertionError(f"{what}: the box test drops a splat that reaches a pixel: splat {vals[s + i]} "
                                 f"record {r[i].tolist()} tile {t[i]} block {b} ({int(miss.sum())} pairs)")
        box_all[sl], poss_all[sl] = box, poss_b
        # the block masks: written for every entry before the tile's largest n_contrib
        before = p[:, None] < nc_tile[t]
        lo, hi = _blocks(certainly & before), _blocks(possibly & before)
        written = p < nc_max[t]
        m = ((strip[sl, None] >> np.arange(8)[None, :]) & 1).astype(bool)
        bad = written[:, None] & ((lo & ~m) | (m & ~hi) | (m & ~box))
        assert not bad.any(), (f"{what}: block mask of {int(bad.any(axis=1).sum())} instances is not the set of blocks "
                               f"its pixels took before n_contrib (first: stream position {s + np.argwhere(bad)[0][0]})")
        cand = possibly & (p[:, None] >= nc_tile[t])
        cp = np.where(cand, p[:, None], np.iinfo(np.int64).max).astype(np.int64)
        np.minimum.at(sat, t, cp)
    # n_contrib never points at a box-dead entry
    hit = nc_tile > 0
    ti, pi = np.nonzero(hit)
    last = ranges[ti, 0].astype(np.int64) + nc_tile[ti, pi] - 1
    assert box_all[last, _BIT[pi]].all(), f"{what}: a pixel's last contributor is box-dead for its block"
    # each block's walk: up to the end of the 32-group in which its last pixel stops (the warp's __all_sync stop)
    stop = np.zeros((len(ranges), 8), np.int64)
    for b in range(8):
        sb = sat[:, _BIT == b].max(axis=1)
        stop[:, b] = np.where(sb < 0, 0, np.minimum(lens, (sb // 32 + 1) * 32))
    walked = pos[:, None] < stop[tile_of]
    return dict(walk=int(walked.sum()), box_skips=int((walked & ~box_all).sum()),
                pixel_skips=int((walked & ~poss_all).sum()))


def _render_scene(sc):
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import rasterizer as R

    R.keep_last_state(True)
    t = {k: sc[k].to(DEV).clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    means2D = torch.zeros((sc["means3D"].shape[0], 3), device=DEV, requires_grad=True)
    g.GaussianRasterizer(h.cuda_settings(sc, DEV), R.FrameHints())(
        means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"], scales=t["scales"],
        rotations=t["rotations"])
    torch.cuda.synchronize()
    return _read_frame(sc["means3D"].shape[0], sc["W"], sc["H"])


MAIN = ["needles", "near_plane", "guard_band", "saturating_stack", "faint", "tile_borders+ties", "guard_band+sh3"]
CASES = [(n, None, None) for n in MAIN] + [(n, W, H) for (W, H) in A.RAGGED_SIZES for n in A.BUILDERS]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0] if c[1] is None else f"{c[0]}-{c[1]}x{c[2]}")
def test_box_cull_on_adversarial_scenes(case):
    from gaussianavatars_b200 import rasterizer as R

    name, W, H = case
    sc = A.saturating_stack(stacks=(20, 400, 2100)) if name == "saturating_stack" and W is None else A.build(name, W, H)
    # the builder's camera, then the rig's narrowed, dollied and mirrored ones: the same splats at other edges
    cams = BR.rig(dict(W=sc["W"], H=sc["H"], cam=sc["cam"], scene=sc), 4)
    try:
        for v, cam in enumerate(cams):
            fr = _render_scene(dict(sc, cam=cam))
            if fr["n"]:
                analyse(fr, f"{name} {sc['W']}x{sc['H']} camera {v}")
    finally:
        R.keep_last_state(False)


def test_box_cull_on_the_headline_frame():
    """bench.py's workload, camera 0: every check, and the fraction of the (block, entry) pairs inside the walk that
    the box skips, beside the fraction a per-pixel exact test would skip."""
    from gaussianavatars_b200 import rasterizer as R
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render

    class Pipe:
        debug = False
        compute_cov3D_python = False
        convert_SHs_python = False

    W, H, P = 1920, 1080, 100_000
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=DEV, requires_grad=True)
    pc.update_mesh_properties(syn.pose_mesh(pc.verts_rest, 0).contiguous())
    cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=-60.0 + 120.0 * 0.5 / 16, elevation_deg=0.0).to(DEV)
    R.keep_last_state(True)
    try:
        render(cam, pc, Pipe, torch.ones(3, device=DEV))
        torch.cuda.synchronize()
        fr = _read_frame(P, W, H)
    finally:
        R.keep_last_state(False)
    assert fr["n"] > 100_000
    c = analyse(fr, "headline frame")
    print(f"[forward cull] {fr['n']} instances; (block, entry) pairs inside the walk {c['walk']}; box test skips "
          f"{c['box_skips']} ({c['box_skips'] / c['walk']:.1%}); a per-pixel exact test would skip {c['pixel_skips']} "
          f"({c['pixel_skips'] / c['walk']:.1%})")
    assert c["box_skips"] <= c["pixel_skips"]
