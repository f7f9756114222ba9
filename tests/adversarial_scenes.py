"""Seeded, deterministic scenes that put the rasterizer at its geometric and numerical edges.

Every builder returns the dict of `helpers.random_scene` (activated CPU float32 tensors, camera, W, H, sh_degree, bg;
no "raw" entry) for an identity-view camera (view space = world space, looking down +z) with a focal length of
`focal` pixels.  Positions and sizes are chosen in PIXELS and depth, then converted, so each builder reaches its
regime at any image size:

    needles           thin 3D splats (axis ratio 1e3), long axis up to about the image width
    near_plane        depths just beyond the 0.2 near plane (radius larger than the image), some exactly at it / below
    guard_band        centres beyond 1.3 tan(fov) whose footprints still reach into the image (clamped-J branch)
    saturating_stack  stacks of opacity >= 0.995 splats (alpha on the 0.99 clamp) that end pixels' walks on T < 1e-4
    faint             opacities at 1/255 (1 +- 1e-3), a few ulp around 1/255 on pixel centres, and below 0.99/255
    tile_borders      sub-pixel splats centred on and around the 16-pixel tile borders
and two modifiers: `with_ties` (duplicated positions: equal depth keys, order by splat id) and `sh3_clamped`
(SH degree 3 with f_dc driving some colours below zero).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from gaussianavatars_b200 import synthetic as syn

F32 = np.float32
RAGGED_SIZES = [(1, 1), (1, 37), (37, 1), (15, 17), (17, 15), (33, 31), (4, 20)]


def camera(W, H, focal):
    fovx = math.degrees(2 * math.atan(W / (2 * focal)))
    fovy = math.degrees(2 * math.atan(H / (2 * focal)))
    return syn.look_at_camera(W, H, fovx, fovy)


def default_focal(W, H):
    return max(24.0, 0.8 * max(W, H))


def pixel_of(cam, W, H, xyz):
    """The oracle's pixel centre of world points (float32 arithmetic in its order; splat_oracle.c preprocess)."""
    M = cam.full_proj_transform.numpy().reshape(16).astype(F32)
    x, y, z = (np.asarray(xyz, F32)[:, k] for k in range(3))
    h0 = M[0] * x + M[4] * y + M[8] * z + M[12]
    h1 = M[1] * x + M[5] * y + M[9] * z + M[13]
    h3 = M[3] * x + M[7] * y + M[11] * z + M[15]
    pw = F32(1.0) / (h3 + F32(0.0000001))
    ndc_x, ndc_y = h0 * pw, h1 * pw
    px = (((ndc_x.astype(np.float64) + 1.0) * W - 1.0) * 0.5).astype(F32)
    py = (((ndc_y.astype(np.float64) + 1.0) * H - 1.0) * 0.5).astype(F32)
    return px, py


def unproject(cam, W, H, u, v, z, exact=False):
    """World points whose pixel centre is (u, v) at view depth z.  exact=True walks x and y by ulps until the oracle's
    float32 pixel centre equals the target exactly (when some float32 position reaches it)."""
    u, v, z = (np.asarray(a, np.float64) for a in (u, v, z))
    tx, ty = cam.tanfovx, cam.tanfovy
    x = ((2 * u + 1) / W - 1) * z * tx
    y = ((2 * v + 1) / H - 1) * z * ty
    xyz = np.stack([x, y, z], 1).astype(F32)
    if exact:
        for k, target in ((0, u.astype(F32)), (1, v.astype(F32))):
            for _ in range(64):
                got = pixel_of(cam, W, H, xyz)[k]
                off = got != target
                if not off.any():
                    break
                step = np.where(got < target, np.inf, -np.inf).astype(F32)
                xyz[off, k] = np.nextafter(xyz[off, k], step[off])
    return xyz


def _rotations(gen, n):
    q = torch.randn(n, 4, generator=gen)
    return q / q.norm(dim=1, keepdim=True)


def _shs(gen, n, deg, dc_lo=-1.0, dc_hi=1.5):
    M = (deg + 1) ** 2
    dc = dc_lo + (dc_hi - dc_lo) * torch.rand(n, 1, 3, generator=gen)
    rest = 0.3 * torch.randn(n, M - 1, 3, generator=gen)
    return torch.cat([dc, rest], 1)


def _scene(cam, W, H, means, scales, rotations, opacities, shs, sh_degree, bg=(0.1, 0.4, 0.8), **extra):
    t = lambda a: torch.as_tensor(np.asarray(a, F32)).contiguous()  # noqa: E731
    sc = dict(means3D=t(means), scales=t(scales), rotations=t(rotations), opacities=t(np.reshape(opacities, (-1, 1))),
              shs=torch.as_tensor(shs, dtype=torch.float32).contiguous(), cam=cam, W=W, H=H, sh_degree=sh_degree,
              bg=torch.tensor(bg, dtype=torch.float32))
    sc.update(extra)
    return sc


def _uniform(gen, n, lo, hi):
    return lo + (hi - lo) * torch.rand(n, generator=gen).numpy().astype(np.float64)


def needles(W=48, H=40, P=80, seed=0, sh_degree=0, focal=None):
    """Scales (s, s 1e-3, s 1e-3) under random rotations, 3 s up to about the image width (in pixels), high opacity."""
    f = focal or default_focal(W, H)
    cam, g = camera(W, H, f), torch.Generator().manual_seed(seed)
    z = _uniform(g, P, 2.0, 5.0)
    xyz = unproject(cam, W, H, _uniform(g, P, -0.2 * W, 1.2 * W), _uniform(g, P, -0.2 * H, 1.2 * H), z)
    sigma_px = _uniform(g, P, 0.05, 0.35) * max(W, H, 8)
    s = sigma_px * z / f
    scales = np.stack([s, s * 1e-3, s * 1e-3], 1)
    opac = _uniform(g, P, 0.6, 0.99)
    return _scene(cam, W, H, xyz, scales, _rotations(g, P), opac, _shs(g, P, sh_degree), sh_degree)


def near_plane(W=48, H=40, P=48, seed=0, sh_degree=0, focal=None):
    """Depths in (0.2, 0.35] with footprints larger than the image; 4 splats at exactly z = 0.2f, 4 one ulp below and
    4 one ulp above; a sparse background at depth 2..4."""
    f = focal or default_focal(W, H)
    cam, g = camera(W, H, f), torch.Generator().manual_seed(seed)
    n_bg = P // 4
    n_near = P - n_bg
    z = np.concatenate([_uniform(g, n_near, 0.2, 0.35), _uniform(g, n_bg, 2.0, 4.0)]).astype(F32)
    z[z <= F32(0.2)] = np.nextafter(F32(0.2), F32(1))
    z02 = F32(0.2)
    z[0:4] = z02
    z[4:8] = np.nextafter(z02, F32(0))
    z[8:12] = np.nextafter(z02, F32(1))
    xyz = unproject(cam, W, H, _uniform(g, P, -1.0 * W, 2.0 * W), _uniform(g, P, -1.0 * H, 2.0 * H), z)
    xyz[:, 2] = z
    near = np.arange(P) < n_near
    # sigma in pixels at that depth: 0.4 .. 1.5 image sizes in front, a few pixels behind
    sigma_px = np.where(near, _uniform(g, P, 0.4, 1.5) * max(W, H, 8), _uniform(g, P, 1.0, 4.0))
    s = sigma_px * z / f
    aniso = np.exp(_uniform(g, 3 * P, -0.5, 0.5)).reshape(P, 3)
    opac = np.where(near, _uniform(g, P, 0.05, 0.5), _uniform(g, P, 0.3, 0.95))
    return _scene(cam, W, H, xyz, s[:, None] * aniso, _rotations(g, P), opac, _shs(g, P, sh_degree), sh_degree)


def guard_band(W=48, H=40, P=48, seed=0, sh_degree=0, focal=None):
    """Centres with |x/z| or |y/z| in (1.3, 3) tan(fov) -- outside the guard band -- with footprints reaching into the
    image; a quarter of them outside in both x and y."""
    f = focal or default_focal(W, H)
    cam, g = camera(W, H, f), torch.Generator().manual_seed(seed)
    tx, ty = cam.tanfovx, cam.tanfovy
    z = _uniform(g, P, 1.0, 3.0)
    side = torch.randint(0, 4, (P,), generator=g).numpy()
    sx = np.where(torch.rand(P, generator=g).numpy() < 0.5, -1.0, 1.0)
    sy = np.where(torch.rand(P, generator=g).numpy() < 0.5, -1.0, 1.0)
    out_x = _uniform(g, P, 1.35, 2.9) * sx
    out_y = _uniform(g, P, 1.35, 2.9) * sy
    in_x = _uniform(g, P, -1.0, 1.0)
    in_y = _uniform(g, P, -1.0, 1.0)
    rx = np.where(side != 1, out_x, in_x)   # side 0: x outside, 1: y outside, 2/3: both
    ry = np.where(side >= 1, out_y, in_y)
    xyz = np.stack([rx * tx * z, ry * ty * z, z], 1).astype(F32)
    # distance to the image in pixels along the clamped axis ~ (|r| - 1) tan(fov) f: a sigma that reaches back in
    reach = np.maximum(np.where(side != 1, (np.abs(rx) - 1) * tx * f, 0), np.where(side >= 1, (np.abs(ry) - 1) * ty * f, 0))
    sigma_px = reach * _uniform(g, P, 0.45, 0.9) + 1.0
    s = sigma_px * z / f
    aniso = np.exp(_uniform(g, 3 * P, -0.4, 0.4)).reshape(P, 3)
    opac = _uniform(g, P, 0.4, 0.99)
    return _scene(cam, W, H, xyz, s[:, None] * aniso, _rotations(g, P), opac, _shs(g, P, sh_degree), sh_degree)


def saturating_stack(W=37, H=33, stacks=(20, 400), seed=0, sh_degree=0, focal=None, opacity=(0.995, 0.999), n_bg=24):
    """Stacks of high-opacity splats (alpha clamped at 0.99 near their centres) at distinct depths, each over a 5x5
    pixel patch that covers part of one tile (saturated and unsaturated pixels in the same tile), over a sparse
    background.  Stack sizes straddle the 32-entry (light/heavy) and 1984/2048-entry blend thresholds when asked."""
    f = focal or default_focal(W, H)
    cam, g = camera(W, H, f), torch.Generator().manual_seed(seed)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    us, vs, zs, sig = [], [], [], []
    for k, n in enumerate(stacks):
        tile = k % (gx * gy)
        # patch inside tile `tile`, offset so that the tile also holds pixels the stack never saturates
        cx = min(16 * (tile % gx) + 5, W - 1)
        cy = min(16 * (tile // gx) + 6, H - 1)
        us.append(cx + _uniform(g, n, -2.5, 2.5))
        vs.append(cy + _uniform(g, n, -2.5, 2.5))
        zs.append(1.5 + 0.5 * k + 4e-4 * np.arange(n))        # distinct float32 depths, interleaved below
        sig.append(_uniform(g, n, 0.8, 2.2))
    u, v, z = (np.concatenate(a) for a in (us, vs, zs))
    sigma_px = np.concatenate(sig)
    ns = u.shape[0]
    u = np.concatenate([u, _uniform(g, n_bg, 0, W)])
    v = np.concatenate([v, _uniform(g, n_bg, 0, H)])
    z = np.concatenate([z, _uniform(g, n_bg, 1.0, 6.0)])
    sigma_px = np.concatenate([sigma_px, _uniform(g, n_bg, 1.0, 5.0)])
    P = ns + n_bg
    perm = torch.randperm(P, generator=g).numpy()    # stack members are not consecutive ids
    u, v, z, sigma_px = u[perm], v[perm], z[perm], sigma_px[perm]
    xyz = unproject(cam, W, H, u, v, z)
    s = sigma_px * z / f
    aniso = np.exp(_uniform(g, 3 * P, -0.3, 0.3)).reshape(P, 3)
    opac = np.concatenate([_uniform(g, ns, *opacity), _uniform(g, n_bg, 0.2, 0.9)])[perm]
    return _scene(cam, W, H, xyz, s[:, None] * aniso, _rotations(g, P), opac, _shs(g, P, sh_degree), sh_degree,
                  n_stack=ns)


def faint(W=48, H=40, P=144, seed=0, sh_degree=0, focal=None):
    """Opacities at 1/255 (1 +- 1e-3), k ulp around float32(1/255) for splats centred exactly on a pixel centre
    (alpha = opacity there, bit for bit), 0.98/255 and 0.5/255 (below the culled binning's margin), and a few
    ordinary splats."""
    f = focal or default_focal(W, H)
    cam, g = camera(W, H, f), torch.Generator().manual_seed(seed)
    thr = F32(1.0) / F32(255.0)
    kinds = np.arange(P) % 6
    opac = np.empty(P, F32)
    walk = (np.arange(P) // 6) % 7 - 3                     # -3 .. 3 ulp
    for i in range(P):
        k = kinds[i]
        if k == 0:
            o = thr
            for _ in range(abs(int(walk[i]))):
                o = np.nextafter(o, F32(np.inf) if walk[i] > 0 else F32(-np.inf))
            opac[i] = o
        elif k == 1:
            opac[i] = thr * F32(1.0 + 1e-3)
        elif k == 2:
            opac[i] = thr * F32(1.0 - 1e-3)
        elif k == 3:
            opac[i] = thr * F32(0.98)
        elif k == 4:
            opac[i] = thr * F32(0.5)
        else:
            opac[i] = F32(0.3 + 0.6 * float(torch.rand(1, generator=g)))
    # integer pixel centres, exact where float32 reaches one (retried at other pixels until it does, for the
    # splats whose alpha must equal their opacity bit for bit)
    z = _uniform(g, P, 2.0, 4.0)
    xyz = np.zeros((P, 3), F32)
    todo = np.ones(P, bool)
    for attempt in range(40):
        n = int(todo.sum())
        u = torch.randint(0, max(W, 1), (n,), generator=g).numpy().astype(np.float64)
        v = torch.randint(0, max(H, 1), (n,), generator=g).numpy().astype(np.float64)
        xyz[todo] = unproject(cam, W, H, u, v, z[todo], exact=True)
        px, py = pixel_of(cam, W, H, xyz)
        todo &= (kinds == 0) & ((px != np.round(px)) | (py != np.round(py)))
        if not todo.any():
            break
    sigma_px = _uniform(g, P, 0.6, 6.0)
    s = sigma_px * z / f
    aniso = np.exp(_uniform(g, 3 * P, -0.5, 0.5)).reshape(P, 3)
    return _scene(cam, W, H, xyz, s[:, None] * aniso, _rotations(g, P), opac, _shs(g, P, sh_degree), sh_degree)


def tile_borders(W=48, H=40, seed=0, sh_degree=0, focal=None, max_splats=400):
    """Sub-pixel splats (radius 2-3) centred at x in {16k - 0.5, 16k, 16k + 2, 16k + 15, 16k + 15.5} (and the same
    for y), every combination, exactly where float32 reaches it."""
    f = focal or default_focal(W, H)
    cam, g = camera(W, H, f), torch.Generator().manual_seed(seed)

    def coords(S):
        out = []
        for k in range(0, (S + 15) // 16 + 1):
            out += [16 * k - 0.5, 16 * k, 16 * k + 2, 16 * k + 15, 16 * k + 15.5]
        return [c for c in out if -1.0 <= c <= S]

    cu, cv = coords(W), coords(H)
    uu, vv = np.meshgrid(np.array(cu), np.array(cv), indexing="ij")
    u, v = uu.reshape(-1), vv.reshape(-1)
    if u.size > max_splats:
        keep = torch.randperm(u.size, generator=g).numpy()[:max_splats]
        u, v = u[keep], v[keep]
    P = u.size
    z = _uniform(g, P, 2.0, 4.0)
    xyz = unproject(cam, W, H, u, v, z, exact=True)
    sigma_px = _uniform(g, P, 0.05, 0.6)
    s = sigma_px * z / f
    aniso = np.exp(_uniform(g, 3 * P, -0.3, 0.3)).reshape(P, 3)
    opac = _uniform(g, P, 0.5, 0.95)
    return _scene(cam, W, H, xyz, s[:, None] * aniso, _rotations(g, P), opac, _shs(g, P, sh_degree), sh_degree)


def with_ties(sc, frac=0.3, seed=1):
    """Append copies of a `frac` share of the splats at the SAME positions (equal depth keys) with their own scale,
    rotation, opacity and colour, then shuffle the ids: equal keys must come out ordered by splat id."""
    g = torch.Generator().manual_seed(seed)
    P = sc["means3D"].shape[0]
    n = max(1, int(frac * P))
    src = torch.randperm(P, generator=g)[:n]
    jit = lambda t, a: (t[src] * torch.exp(a * torch.randn(t[src].shape, generator=g))).contiguous()  # noqa: E731
    means = torch.cat([sc["means3D"], sc["means3D"][src]])
    scales = torch.cat([sc["scales"], jit(sc["scales"], 0.3)])
    rots = torch.cat([sc["rotations"], _rotations(g, n)])
    opac = torch.cat([sc["opacities"], sc["opacities"][torch.randperm(P, generator=g)[:n]]])
    shs = torch.cat([sc["shs"], sc["shs"][torch.randperm(P, generator=g)[:n]]])
    perm = torch.randperm(P + n, generator=g)
    out = dict(sc)
    out.update(means3D=means[perm].contiguous(), scales=scales[perm].contiguous(), rotations=rots[perm].contiguous(),
               opacities=opac[perm].contiguous(), shs=shs[perm].contiguous())
    out.pop("n_stack", None)
    return out


def sh3_clamped(sc, seed=2):
    """The same geometry at SH degree 3, f_dc in [-2.5, 1]: a good share of the colours clamps at zero."""
    g = torch.Generator().manual_seed(seed)
    P = sc["means3D"].shape[0]
    out = dict(sc)
    out.update(shs=_shs(g, P, 3, dc_lo=-2.5, dc_hi=1.0).contiguous(), sh_degree=3)
    return out


def pair_table(st):
    """Every (sorted instance, pixel of its tile) pair of an oracle forward state, with the blend's own float32
    quantities: instance index j (stream position), splat id, pixel, power, alpha = min(.99, o exp(power)) and
    `live` (j lies before the pixel's n_contrib: the walk had not stopped).  Returns a dict of flat numpy arrays."""
    W, H = st.W, st.H
    gx = (W + 15) // 16
    out = {k: [] for k in ("j", "id", "pix", "power", "alpha", "live")}
    ly, lx = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
    for tile in range(st.ranges.shape[0]):
        r0, r1 = int(st.ranges[tile, 0]), int(st.ranges[tile, 1])
        if r1 <= r0:
            continue
        xs, ys = (tile % gx) * 16 + lx.reshape(-1), (tile // gx) * 16 + ly.reshape(-1)
        inside = (xs < W) & (ys < H)
        xs, ys = xs[inside], ys[inside]
        pix = ys * W + xs
        ids = st.vals_sorted[r0:r1].astype(np.int64)
        co = st.conic_opacity[ids]
        dx = st.xy[ids, 0][:, None] - xs[None, :].astype(F32)
        dy = st.xy[ids, 1][:, None] - ys[None, :].astype(F32)
        power = F32(-0.5) * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
        alpha = np.minimum(F32(0.99), co[:, 3:4] * np.exp(np.minimum(power, F32(0))))
        j = np.arange(r0, r1)[:, None]
        live = (j - r0) < st.n_contrib.reshape(-1)[pix][None, :].astype(np.int64)
        out["j"].append(np.broadcast_to(j, power.shape).reshape(-1))
        out["id"].append(np.broadcast_to(ids[:, None], power.shape).reshape(-1))
        out["pix"].append(np.broadcast_to(pix[None, :], power.shape).reshape(-1))
        out["power"].append(power.reshape(-1))
        out["alpha"].append(alpha.reshape(-1))
        out["live"].append(live.reshape(-1))
    return {k: (np.concatenate(v) if v else np.zeros(0)) for k, v in out.items()}


ALPHA_MIN = F32(1.0) / F32(255.0)


# Error bound of the blend's float32 decisions against the oracle's (the margins of `knife_edges`).  The blend takes
#   pw = fma(C' dy, dy, fma(B', dy, A' dx) dx)   with (A', B', C') = (-A/2, -B, -C/2) log2(e) from its own preprocess,
#   G  = ex2.approx(pw),   alpha = min(.99, o G),
# where the oracle takes power = -(A dx^2 + C dy^2)/2 - B dx dy and G = expf(power).  Per pair, with
#   Q = |A| dx^2/2 + |B dx dy| + |C| dy^2/2   (the terms of the quadratic form, before they cancel):
#   |pw / log2(e) - power| <= KNIFE_CONIC_REL Q        a conic off by up to 128 ulp per component (A and C
#                                                      relative to themselves, B to sqrt|A C|: the exponent then
#                                                      moves by at most twice that times Q).  Measured by
#                                                      tests/test_gpu_preprocess.py: on the plain route the device
#                                                      record is the oracle's bit for bit; on the mesh-bound route,
#                                                      whose activation is the kernel's own rather than the eager
#                                                      getters', the worst component outside the KNIFE_COND class
#                                                      was 112 x 2^-24 (H100 80GB HBM3, 700 W).  A device conic
#                                                      further off shows as unexplained entries, not as a pass;
#   |G'/G - 1| <= that + KNIFE_EXP_REL                 ex2.approx.ftz.f32 is within 2^-22 relative (PTX ISA), expf
#                                                      within one ulp, and o G rounds once.
# At a splat's exact centre (dx = dy = 0) both sides evaluate power = 0 and G = 1 exactly, so alpha = o bit for bit.
KNIFE_CONIC_REL = 2.0 ** -16
KNIFE_EXP_REL = 2.0 ** -20
# A second class, not a decision: a splat whose 3D covariance has condition number kappa carries float32 rounding
# amplified by about kappa through the covariance and conic chain (forward and backward), so the kernel's and the
# oracle's gradients of it may differ by ~kappa 2^-24 relative.  Beyond KNIFE_COND that reaches a tenth of the
# gradient gate's rtol: a needle with axis ratio 1e3 (kappa 1e6) moved one dL/dmeans3D entry by 1.3 % on the H100.
KNIFE_COND = 1e-4 * 2.0 ** 24
T_STOP = F32(0.0001)


def knife_edges(st, conic_rel=KNIFE_CONIC_REL, exp_rel=KNIFE_EXP_REL, xy_abs=0.0):
    """Where a blend whose decisions are within the error bound above of the oracle's may decide otherwise.

    From the float32 oracle state, per (instance, pixel) pair of every tile:
      * knife pairs: `power` within the bound of 0, or `alpha` within it of 1/255 (accepted on one side, skipped on
        the other);
      * the walk under the oracle's decisions: T after each accepted pair (float32, the blend's order) with a relative
        error bound that sums, over the accepted pairs in front, alpha/(1-alpha) times their alpha's error (zero where
        o G clears the 0.99 clamp by the bound) plus one rounding, and alpha/(1-alpha) in full for every knife pair (a
        flip multiplies T by 1-alpha or its inverse).  A pair is REACHED unless an accepted pair in front ends the
        walk (T < 1e-4) by more than that bound;
      * knife pixels: a reached knife pair, or a reached accepted pair whose T is within its bound of 1e-4.
    A flip in a knife pixel moves T for the splats behind it and the colour composited behind the splats in front of
    it, so every splat with a reached accepted or knife pair in a knife pixel is affected.

    `xy_abs` bounds the error of the pixel-space centre (0 when both sides share the preprocess's float32 centre;
    float64 models pass their own).  Returns a dict: `pixels` (H, W) and `splats` (P,) boolean masks, `pairs` (number
    of knife pairs; `ill`, the splats of the KNIFE_COND class, which `affected` adds for the covariance chain's
    gradients only), and the oracle's own `n_contrib` and `final_T` restated from the walk (a check of the restatement).
    """
    W, H = st.W, st.H
    gx = (W + 15) // 16
    pixels = np.zeros(H * W, bool)
    splats = np.zeros(st.P, bool)
    n_contrib = np.zeros(H * W, np.int64)
    final_T = np.ones(H * W, F32)
    n_pairs = 0
    ly, lx = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
    for tile in range(st.ranges.shape[0]):
        r0, r1 = int(st.ranges[tile, 0]), int(st.ranges[tile, 1])
        if r1 <= r0:
            continue
        xs, ys = (tile % gx) * 16 + lx.reshape(-1), (tile // gx) * 16 + ly.reshape(-1)
        inside = (xs < W) & (ys < H)
        xs, ys = xs[inside], ys[inside]
        pix = ys * W + xs
        ids = st.vals_sorted[r0:r1].astype(np.int64)
        co = st.conic_opacity[ids]
        dx = st.xy[ids, 0][:, None] - xs[None, :].astype(F32)
        dy = st.xy[ids, 1][:, None] - ys[None, :].astype(F32)
        power = F32(-0.5) * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
        og = co[:, 3:4] * np.exp(np.minimum(power, F32(0)).astype(np.float64)).astype(F32)   # expf, correctly rounded
        alpha = np.minimum(F32(0.99), og)
        acc = (power <= 0) & (alpha >= ALPHA_MIN)
        A, B, C = (co[:, k:k + 1].astype(np.float64) for k in range(3))
        dx64, dy64 = dx.astype(np.float64), dy.astype(np.float64)
        Q = 0.5 * np.abs(A) * dx64 ** 2 + np.abs(B * dx64 * dy64) + 0.5 * np.abs(C) * dy64 ** 2
        dpow = conic_rel * Q + xy_abs * (np.abs(A * dx64 + B * dy64) + np.abs(B * dx64 + C * dy64))
        rel = np.where(Q == 0, 0.0, dpow + exp_rel)          # relative error bound of G, hence of o G
        a64 = alpha.astype(np.float64)
        knife = ((Q > 0) & (np.abs(power) <= dpow)) | ((power <= dpow) & (np.abs(a64 - float(ALPHA_MIN)) < a64 * rel))
        odds = a64 / (1.0 - a64)
        firm = og.astype(np.float64) * (1.0 - rel) >= 0.99   # on the clamp on both sides
        d = np.where(acc, np.where(firm, 0.0, odds * rel) + 2.0 ** -23, 0.0) + np.where(knife, odds, 0.0)
        T = np.cumprod(np.where(acc, F32(1) - alpha, F32(1)), axis=0, dtype=F32)   # T after each pair
        margin = T.astype(np.float64) * np.expm1(np.cumsum(d, axis=0))
        ends = acc & (T.astype(np.float64) + margin < float(T_STOP))
        reached = np.cumsum(ends, axis=0) - ends == 0        # no accepted pair in front ends the walk for sure
        near_stop = acc & reached & (np.abs(T.astype(np.float64) - float(T_STOP)) <= margin)
        kpix = (knife & reached).any(0) | near_stop.any(0)
        pixels[pix] |= kpix
        hit = ((acc | knife) & reached)[:, kpix].any(1)
        splats[ids[hit]] = True
        n_pairs += int((knife & reached).sum())
        # the oracle's walk itself: it stops at the first accepted pair that takes T below 1e-4
        stop = acc & (T < T_STOP)
        live = np.cumsum(stop, axis=0) == 0
        took = acc & live
        last = np.where(took.any(0), took.shape[0] - np.argmax(took[::-1], axis=0), 0)
        n_contrib[pix] = last
        final_T[pix] = np.where(took.any(0), T[np.maximum(last - 1, 0), np.arange(pix.size)], F32(1))
    return dict(pixels=pixels.reshape(H, W), splats=splats, ill=ill_conditioned(st), pairs=n_pairs,
                n_contrib=n_contrib.reshape(H, W), final_T=final_T.reshape(H, W))


def ill_conditioned(st):
    """(P,) the rendered splats of the KNIFE_COND class: 3D covariance condition number beyond KNIFE_COND."""
    c = st.cov3D.astype(np.float64)
    S = np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], 1)
    ev = np.abs(np.linalg.eigvalsh(S))
    return (st.radii > 0) & (ev[:, 2] > KNIFE_COND * ev[:, 0])


# the gradients that pass through the covariance and conic chain of the preprocess (activated and bound names)
COV_CHAIN = {"means3D", "scales", "rotations", "cov3D_precomp", "_xyz", "_scaling", "_rotation"}


def affected(ke, name):
    """The splats knife_edges explains for the gradient `name`: the knife splats, and for the tensors of the
    covariance chain also the ill-conditioned ones (the blend's own outputs -- means2D, opacity, colour -- do not
    pass through that chain, so no condition number explains an error in them)."""
    return ke["splats"] | ke["ill"] if name in COV_CHAIN else ke["splats"]


def accepted_instances(st):
    """Stream positions j the oracle's blend took into some pixel (power <= 0, alpha >= 1/255, before n_contrib)."""
    t = pair_table(st)
    acc = (t["power"] <= 0) & (t["alpha"] >= ALPHA_MIN) & t["live"]
    return np.unique(t["j"][acc])


BUILDERS = dict(needles=needles, near_plane=near_plane, guard_band=guard_band, saturating_stack=saturating_stack,
                faint=faint, tile_borders=tile_borders)


def build(name, W=None, H=None, seed=0, **kw):
    """Builder by name; "X+ties" appends duplicated positions; "X+sh3" switches to the clamping SH-3 colours."""
    base, *mods = name.split("+")
    size = {} if W is None else dict(W=W, H=H)
    sc = BUILDERS[base](seed=seed, **size, **kw)
    for m in mods:
        sc = {"ties": with_ties, "sh3": sh3_clamped}[m](sc)
    sc["name"] = name
    return sc
