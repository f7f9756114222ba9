"""Seeded scenes that put the per-splat preprocess at each of its edges, one family of splats per regime, and a float32
restatement of the oracle's projection that says which regime every splat reached.

Every scene is the dict of `helpers.random_scene` (activated CPU float32 tensors, an identity-view camera looking down
+z from adversarial_scenes.camera, W, H, sh_degree) plus `family`, the (P,) array of family names (failure messages
name a splat's family), and `scale_modifier`.  The families:

    guard        centres at x/z, y/z = +-1.3 tan(fov) and a few ulp either side of it, corners, far outside
    near         depth 0.2 and a few ulp either side; depths just beyond it with radii far beyond the image
    needle       axis ratios 1e2 .. 1e4, long axis in the image plane (face-on) or along the view ray (edge-on)
    radius_edge  isotropic splats swept by ulps of their scale across 3 sqrt(lambda_max) = integer, centred on tile
                 borders
    offscreen    centres left of / above the image at a distance around their radius: some reach in, some miss by a
                 tile
    scale        scales from 1e-7 to 1e3 (log-uniform), mildly anisotropic
    quat         quaternions of norm 1e-3 and 1e3, and with w < 0
    colour       SH sums a few ulp below, at and above the 0 clamp of each channel; view directions with zero
                 components (on the view axis and the coordinate planes)
    plain        ordinary splats in front of the camera

`edge_scene(...)` also takes the colors_precomp and cov3D_precomp routes.  `regimes(sc, st)` counts, per regime, the
splats of an oracle forward state that reached it; test_oracle_preprocess.py asserts that every one is reached.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import adversarial_scenes as A

F32 = np.float32


def _ulps(x, k):
    """x moved k ulps (k may be negative), elementwise, float32."""
    x, k = np.broadcast_arrays(np.asarray(x, F32), np.asarray(k))
    x = x.copy()
    for j in range(int(np.abs(k).max()) if k.size else 0):
        step = np.abs(k) > j
        x[step] = np.nextafter(x[step], np.where(k[step] > 0, F32(np.inf), F32(-np.inf)).astype(F32))
    return x


def _unit_quats(g, n):
    q = torch.randn(n, 4, generator=g)
    return (q / q.norm(dim=1, keepdim=True)).numpy()


def edge_scene(W=160, H=120, seed=0, sh_degree=3, max_sh_degree=3, scale_modifier=1.0, route="shs"):
    """All families in one scene, about 2.5k splats.  route: "shs" (SH colours, scale / rotation), "colors_precomp"
    or "cov3D_precomp" (the same splats through those inputs)."""
    f = A.default_focal(W, H)
    cam = A.camera(W, H, f)
    g = torch.Generator().manual_seed(seed)
    tx, ty = F32(cam.tanfovx), F32(cam.tanfovy)
    u = lambda n, lo, hi: (lo + (hi - lo) * torch.rand(n, generator=g).numpy()).astype(np.float64)  # noqa: E731
    fam, xyz, sc, rot, op = [], [], [], [], []

    def add(name, p, s, q=None, o=None):
        n = p.shape[0]
        fam.extend([name] * n)
        xyz.append(np.asarray(p, F32))
        sc.append(np.asarray(s, F32))
        rot.append(np.asarray(_unit_quats(g, n) if q is None else q, F32))
        op.append(np.asarray(u(n, 0.3, 0.95) if o is None else o, F32))

    # guard: t.x / t.z within k ulps of +-limx (float32, as the preprocess forms the ratio), and the same in y
    lim = (F32(1.3) * tx, F32(1.3) * ty)
    for axis in (0, 1):
        k = np.repeat(np.arange(-4, 5), 8)
        n = k.size
        z = u(n, 1.0, 3.0).astype(F32)
        sign = np.where(np.arange(n) % 2 == 0, F32(1), F32(-1))
        r = _ulps(lim[axis], k) * sign
        p = np.zeros((n, 3), F32)
        p[:, 2] = z
        p[:, axis] = r * z
        # walk the coordinate until the float32 ratio is the target exactly (or its neighbour)
        for _ in range(8):
            got = p[:, axis] / p[:, 2]
            off = got != r
            p[off, axis] = np.nextafter(p[off, axis], np.where(got[off] < r[off], F32(np.inf), F32(-np.inf)))
        p[:, 1 - axis] = (u(n, -0.8, 0.8) * float([tx, ty][1 - axis]) * z).astype(F32)
        sig = 0.3 * float([tx, ty][axis]) * f * u(n, 0.5, 1.2) + 1.0
        add("guard", p, (sig * z / f)[:, None] * np.exp(u(3 * n, -0.3, 0.3)).reshape(n, 3))
    # corners and far outside, both axes
    n = 64
    z = u(n, 1.0, 3.0)
    rx = u(n, 1.31, 12.0) * np.where(np.arange(n) % 2 == 0, 1, -1)
    ry = u(n, 1.31, 12.0) * np.where((np.arange(n) // 2) % 2 == 0, 1, -1)
    p = np.stack([rx * float(tx) * z, ry * float(ty) * z, z], 1)
    sig = (np.maximum(np.abs(rx) - 1, 0) * float(tx) * f) * u(n, 0.4, 1.1) + 2.0
    add("guard", p, (sig * z / f)[:, None] * np.exp(u(3 * n, -0.3, 0.3)).reshape(n, 3))

    # near: z = 0.2 and k ulps either side; just in front with radii many times the image
    k = np.repeat(np.arange(-3, 4), 6)
    n = k.size
    z = _ulps(np.full(n, F32(0.2)), k)
    p = np.stack([u(n, -0.5, 0.5) * float(tx) * z, u(n, -0.5, 0.5) * float(ty) * z, z], 1).astype(F32)
    p[:, 2] = z
    add("near", p, (u(n, 1.0, 4.0) * max(W, H) * z / f)[:, None] * np.ones((1, 3)))
    n = 48
    z = u(n, 0.2005, 0.26)
    p = np.stack([u(n, -1.2, 1.2) * float(tx) * z, u(n, -1.2, 1.2) * float(ty) * z, z], 1)
    add("near", p, (u(n, 2.0, 10.0) * max(W, H) * z / f)[:, None] * np.exp(u(3 * n, -0.5, 0.5)).reshape(n, 3),
        o=u(n, 0.02, 0.3))

    # needles: long axis in the image plane (x: face-on) or along the view ray (z: edge-on)
    for ratio in (1e2, 1e3, 1e4):
        for long_axis in (0, 2):
            n = 40
            z = u(n, 2.0, 5.0)
            p = A.unproject(cam, W, H, u(n, 0.0, W), u(n, 0.0, H), z)
            s_long = u(n, 0.05, 0.3) * max(W, H) * z / f
            s = np.repeat((s_long / ratio)[:, None], 3, 1)
            s[:, long_axis] = s_long
            q = np.tile(np.array([1.0, 0.0, 0.0, 0.0]), (n, 1))
            q[n // 2:] = _unit_quats(g, n - n // 2) * np.array([1.0, 1e-3, 1e-3, 1e-3])   # nearly aligned
            q[n // 2:] /= np.linalg.norm(q[n // 2:], axis=1, keepdims=True)
            add("needle", p, s, q)

    # radius_edge: isotropic splats on tile borders whose 3 sqrt(lambda_max) is an integer m to within an ulp, found
    # by bisection in float64 and a sweep of the scale's ulps through the float32 restatement, with the scales one ulp
    # either side of the best one
    V, Pm = cam.world_view_transform.numpy(), cam.full_proj_transform.numpy()
    mm = np.repeat(np.arange(2, 42, 2), 4).astype(np.float64)
    n = mm.size
    gxn, gyn = max(1, W // 16 - 1), max(1, H // 16 - 1)
    us = 16.0 * (1 + np.arange(n) % gxn)
    vs = 16.0 * (1 + (np.arange(n) * 7) % gyn) + np.where(np.arange(n) % 4 == 3, 0.5, 0.0)
    z = u(n, 2.0, 4.0)
    p = A.unproject(cam, W, H, us, vs, z, exact=True)
    mod = F32(scale_modifier)

    def r3_of(s32):
        se = mod * np.asarray(s32, F32)
        ss = se * se
        zero = np.zeros_like(ss)
        cov = np.stack([ss, zero, zero, ss, zero, ss], -1).reshape(-1, 6)
        pp = np.repeat(p, s32.shape[1] if s32.ndim > 1 else 1, axis=0)
        return f32_project(pp, V, Pm, W, H, cam.tanfovx, cam.tanfovy, cov)["r3"].reshape(s32.shape)

    lo, hi = np.full(n, 1e-6), np.full(n, 10.0)
    for _ in range(80):
        mid_ = np.sqrt(lo * hi)
        big = r3_of(mid_.astype(F32)[:, None])[:, 0] > mm
        hi, lo = np.where(big, mid_, hi), np.where(big, lo, mid_)
    ks = np.arange(-24, 25)
    cand = _ulps(np.repeat(hi.astype(F32)[:, None], ks.size, 1), np.broadcast_to(ks, (n, ks.size)))
    best = cand[np.arange(n), np.argmin(np.abs(r3_of(cand) - mm[:, None]), axis=1)]
    s = np.concatenate([_ulps(best, d) for d in (-1, 0, 1)])
    add("radius_edge", np.tile(p, (3, 1)), np.repeat(s[:, None], 3, 1), np.tile([1.0, 0.0, 0.0, 0.0], (3 * n, 1)))

    # offscreen: centre left of / above the image, the gap to the image edge swept around the radius
    n = 96
    z = u(n, 1.5, 3.0)
    sig = u(n, 3.0, 12.0)
    gap = 3.0 * sig + np.linspace(-40.0, 12.0, n)             # px = -gap: reaches in for gap < radius
    side = np.arange(n) % 2
    px = np.where(side == 0, -gap, u(n, 0, W))
    py = np.where(side == 1, -gap, u(n, 0, H))
    p = A.unproject(cam, W, H, px, py, z)
    add("offscreen", p, (sig * z / f)[:, None] * np.ones((1, 3)), np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)))

    # scale: 1e-7 .. 1e3 (log-uniform per splat; the anisotropy is the needles' business)
    n = 160
    z = u(n, 2.0, 6.0)
    p = A.unproject(cam, W, H, u(n, 0.0, W), u(n, 0.0, H), z)
    s = (10.0 ** u(n, -7.0, 3.0))[:, None] * np.exp(u(3 * n, -1.0, 1.0)).reshape(n, 3)
    add("scale", p, s, o=u(n, 0.05, 0.9))

    # quat: norm 1e-3 and 1e3 (scales shrunk so that the footprint stays image-sized), w < 0
    n = 120
    z = u(n, 2.0, 5.0)
    p = A.unproject(cam, W, H, u(n, 0.0, W), u(n, 0.0, H), z)
    q = _unit_quats(g, n)
    norm = np.where(np.arange(n) % 3 == 0, 1e-3, np.where(np.arange(n) % 3 == 1, 1e3, 1.0))
    q[:, 0] = -np.abs(q[:, 0])
    q = q * norm[:, None]
    sig = u(n, 1.0, 8.0)
    s_eff = np.where(norm > 1, 1.0 / (norm * norm), 1.0)       # R(q) grows as |q|^2
    add("quat", p, (sig * z / f * s_eff)[:, None] * np.exp(u(3 * n, -0.4, 0.4)).reshape(n, 3), q)

    # colour: splats whose SH sum sits a few ulp from 0 (coefficients beyond the DC set to 0 for them, below), and
    # view directions with zero components
    n_col = 3 * 9
    z = u(n_col, 2.0, 4.0)
    p = A.unproject(cam, W, H, u(n_col, 0.0, W), u(n_col, 0.0, H), z)
    add("colour", p, (u(n_col, 1.0, 6.0) * z / f)[:, None] * np.ones((1, 3)))
    n_ax = 24
    z = u(n_ax, 1.0, 4.0)
    p = np.stack([np.where(np.arange(n_ax) % 3 != 1, 0.0, u(n_ax, -0.3, 0.3) * z),
                  np.where(np.arange(n_ax) % 3 != 2, 0.0, u(n_ax, -0.3, 0.3) * z), z], 1)
    add("colour", p, (u(n_ax, 1.0, 6.0) * z / f)[:, None] * np.ones((1, 3)))

    # plain: the bulk
    n = 1200
    z = u(n, 1.5, 8.0)
    p = A.unproject(cam, W, H, u(n, -0.1 * W, 1.1 * W), u(n, -0.1 * H, 1.1 * H), z)
    add("plain", p, (u(n, 0.3, 8.0) * z / f)[:, None] * np.exp(u(3 * n, -0.7, 0.7)).reshape(n, 3))

    family = np.array(fam)
    P = family.size
    means = np.concatenate(xyz).astype(F32)
    scales = np.concatenate(sc).astype(F32)
    rots = np.concatenate(rot).astype(F32)
    opac = np.concatenate(op).astype(F32).reshape(P, 1)
    M = (max_sh_degree + 1) ** 2
    shs = np.zeros((P, M, 3), F32)
    shs[:, 0] = u(3 * P, -1.0, 1.5).reshape(P, 3)
    shs[:, 1:] = 0.3 * torch.randn(P, M - 1, 3, generator=g).numpy()
    # colour family: channel ch of splat j has rgb = C0 dc + 0.5 a few ulp off 0 (the other coefficients are 0)
    col = np.nonzero(family == "colour")[0][:n_col]
    dc0 = F32(-0.5) / F32(0.28209479177387814)
    for j, i in enumerate(col):
        shs[i, 1:] = 0.0
        shs[i, 0, :] = F32(0.3)
        shs[i, 0, j % 3] = _ulps(np.array([dc0]), np.array([j // 3 - 4]))[0]
    sc_ = dict(means3D=torch.from_numpy(means), scales=torch.from_numpy(scales), rotations=torch.from_numpy(rots),
               opacities=torch.from_numpy(opac), shs=torch.from_numpy(shs), cam=cam, W=W, H=H, sh_degree=sh_degree,
               bg=torch.tensor([0.1, 0.4, 0.8]), family=family, scale_modifier=float(scale_modifier), route=route)
    if route == "colors_precomp":
        sc_["colors_precomp"] = torch.from_numpy(u(3 * P, -0.2, 1.2).reshape(P, 3).astype(F32))
    elif route == "cov3D_precomp":
        sc_["cov3D_precomp"] = torch.from_numpy(cov3d_f64(scales.astype(np.float64) * scale_modifier, rots).astype(F32))
    elif route != "shs":
        raise ValueError(route)
    return sc_


def cov3d_f64(s, q):
    """(P,6) Sigma = R(q) diag(s^2) R(q)^T in float64, q used as given."""
    from oracle import dense64

    R = dense64.quat_to_R(torch.as_tensor(q, dtype=torch.float64)).numpy()
    S = np.einsum("pik,pk,pjk->pij", R, np.asarray(s, np.float64) ** 2, R)
    return np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)


def oracle_kwargs(sc):
    """The keyword arguments of oracle.rasterizer.forward for the scene's route."""
    kw = dict(sh_degree=sc["sh_degree"], scale_modifier=sc["scale_modifier"])
    if "colors_precomp" in sc:
        kw["colors_precomp"] = sc["colors_precomp"].numpy()
    else:
        kw["shs"] = sc["shs"].numpy()
    if "cov3D_precomp" in sc:
        kw["cov3D_precomp"] = sc["cov3D_precomp"].numpy()
    else:
        kw.update(scales=sc["scales"].numpy(), rotations=sc["rotations"].numpy())
    return kw


def f32_project(means3D, V, Pm, W, H, tanfovx, tanfovy, cov3D):
    """The oracle's projection restated in numpy float32, operation for operation (no contraction): view-space t,
    the guard-band clamp bits (P,2), the dilated 2-D covariance, det, 3 sqrt(lambda_max), the radius and
    `conic_dropped` (the backward's 1 / (det^2 + 1e-7) is 0: no gradient through the conic).  `cov3D`
    (P,6) float32: the oracle state's cov3D."""
    m = np.asarray(means3D, F32)
    V = np.asarray(V, F32).reshape(16)
    x, y, z = m[:, 0], m[:, 1], m[:, 2]
    t = [V[r] * x + V[4 + r] * y + V[8 + r] * z + V[12 + r] for r in range(3)]
    tanfovx, tanfovy = F32(tanfovx), F32(tanfovy)
    fx, fy = F32(W) / (F32(2) * tanfovx), F32(H) / (F32(2) * tanfovy)
    limx, limy = F32(1.3) * tanfovx, F32(1.3) * tanfovy
    with np.errstate(all="ignore"):
        txtz, tytz = t[0] / t[2], t[1] / t[2]
        guard = np.stack([(txtz < -limx) | (txtz > limx), (tytz < -limy) | (tytz > limy)], 1)
        tcx = np.minimum(limx, np.maximum(-limx, txtz)) * t[2]
        tcy = np.minimum(limy, np.maximum(-limy, tytz)) * t[2]
        j00, j02 = fx / t[2], -(fx * tcx) / (t[2] * t[2])
        j11, j12 = fy / t[2], -(fy * tcy) / (t[2] * t[2])
        T0 = [j00 * V[4 * c] + j02 * V[4 * c + 2] for c in range(3)]
        T1 = [j11 * V[4 * c + 1] + j12 * V[4 * c + 2] for c in range(3)]
        c3 = np.asarray(cov3D, F32)
        S = [c3[:, k] for k in (0, 1, 2, 1, 3, 4, 2, 4, 5)]
        uu = [S[3 * i] * T0[0] + S[3 * i + 1] * T0[1] + S[3 * i + 2] * T0[2] for i in range(3)]
        vv = [S[3 * i] * T1[0] + S[3 * i + 1] * T1[1] + S[3 * i + 2] * T1[2] for i in range(3)]
        a = T0[0] * uu[0] + T0[1] * uu[1] + T0[2] * uu[2] + F32(0.3)
        b = T0[0] * vv[0] + T0[1] * vv[1] + T0[2] * vv[2]
        c = T1[0] * vv[0] + T1[1] * vv[1] + T1[2] * vv[2] + F32(0.3)
        det = a * c - b * b
        mid = F32(0.5) * (a + c)
        sq = np.sqrt(np.where(F32(0.1) > mid * mid - det, F32(0.1), mid * mid - det))
        lam = np.where(mid + sq > mid - sq, mid + sq, mid - sq)
        r3 = F32(3) * np.sqrt(lam)
        conic_dropped = F32(1) / (det * det + F32(0.0000001)) == 0   # the backward's guard: det^2 overflows
    return dict(t=np.stack(t, 1), guard=guard, cov2d=np.stack([a, b, c], 1), det=det, r3=r3, radius=np.ceil(r3),
                conic_dropped=conic_dropped)


def regimes(sc, st):
    """{regime: (P,) bool} of the splats of oracle state `st` (of scene `sc`) that reached it."""
    cam, W, H = sc["cam"], sc["W"], sc["H"]
    pr = f32_project(sc["means3D"].numpy(), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(), W, H,
                     cam.tanfovx, cam.tanfovy, st.cov3D)
    kept = st.radii > 0
    tz = pr["t"][:, 2]
    lim = np.array([F32(1.3) * F32(cam.tanfovx), F32(1.3) * F32(cam.tanfovy)], F32)
    with np.errstate(all="ignore"):
        ratio = np.abs(pr["t"][:, :2] / pr["t"][:, 2:3])
    ulp = np.spacing(lim)[None, :]
    near_lim = np.abs(ratio - lim[None, :]) <= 4 * ulp
    r3 = pr["r3"]
    out = {
        "guard x clamped": kept & pr["guard"][:, 0], "guard y clamped": kept & pr["guard"][:, 1],
        "guard both clamped": kept & pr["guard"].all(1),
        "guard ratio ulps above the limit": kept & near_lim.any(1) & pr["guard"].any(1),
        "guard ratio ulps below or at the limit": kept & (near_lim & ~pr["guard"]).any(1),
        "near plane cull at z <= 0.2": (tz <= F32(0.2)) & (tz > F32(0.2) * F32(0.99999)),
        "kept one ulp beyond z = 0.2": kept & (tz <= np.nextafter(F32(0.2), F32(1), dtype=F32) * F32(1.000001)),
        "radius beyond the image": kept & (st.radii > 2 * max(W, H)),
        "conic gradient dropped (det^2 overflows)": kept & pr["conic_dropped"],
        "needle (KNIFE_COND)": A.ill_conditioned(st),
        "3 sqrt(lambda) within an ulp of an integer": kept & (np.abs(r3 - np.round(r3)) <= np.spacing(r3)),
        "centre on a tile border": kept & ((st.xy[:, 0] % 16 == 0) | (st.xy[:, 1] % 16 == 0)),
        "centre off-screen, radius reaches in": kept & ((st.xy[:, 0] < -1) | (st.xy[:, 1] < -1)),
        "off-screen, misses the image": (tz > F32(0.2)) & (pr["det"] != 0) & ~kept,
        "scale below 1e-5": kept & (sc["scales"].numpy().max(1) < 1e-5),
        "scale above 1e2": kept & (sc["scales"].numpy().max(1) > 1e2),
        "quaternion norm 1e-3": kept & (np.linalg.norm(sc["rotations"].numpy(), axis=1) < 1e-2),
        "quaternion norm 1e3": kept & (np.linalg.norm(sc["rotations"].numpy(), axis=1) > 1e2),
        "quaternion w < 0": kept & (sc["rotations"].numpy()[:, 0] < 0),
    }
    if "colors_precomp" not in sc:
        for ch in range(3):
            out[f"colour channel {ch} clamped"] = kept & (st.clamped[:, ch] != 0)
        out["colour within 1e-6 above the clamp"] = kept & ((st.rgb >= 0) & (st.rgb < 1e-6) & (st.clamped == 0)).any(1)
        d = sc["means3D"].numpy() - cam.camera_center.numpy()[None, :]
        out["view direction with a zero component"] = kept & (d == 0).any(1)
    return out


# --------------------------------------------------------------------------------------------------------------------
# The per-splat upstream of the preprocess backward and its three consumers
# --------------------------------------------------------------------------------------------------------------------
# g2d row (GAB_G2D_STRIDE floats per splat, csrc/common.cuh): dL/dndc.xy, dL/dconic (A, B stored once, C), dL/dopacity,
# dL/drgb, dL/dz (the depth plane), 2 unused
G2D = 12
FIELDS = {"ndc": (0, 2), "conic": (2, 5), "opacity": (5, 6), "rgb": (6, 9), "z": (9, 10)}
PLAIN_INPUTS = ("means3D", "scales", "rotations", "shs", "opacities", "cov3D_precomp", "colors_precomp")


def upstream(P, kind, seed=0, with_z=False):
    """(P, 12) float32 per-splat upstream: "random" (every field), "zero", or "one-hot:<field>" (that field only)."""
    g = torch.Generator().manual_seed(seed)
    up = torch.randn(P, G2D, generator=g).numpy().astype(F32)
    up[:, 10:] = 0
    if not with_z:
        up[:, 9] = 0
    if kind == "zero":
        up[:] = 0
    elif kind.startswith("one-hot:"):
        lo, hi = FIELDS[kind.split(":")[1]]
        keep = np.zeros(G2D, bool)
        keep[lo:hi] = True
        up[:, ~keep] = 0
    return up


def cam_args(sc):
    cam = sc["cam"]
    return (cam.world_view_transform.double(), cam.full_proj_transform.double(), cam.camera_center.double(), sc["W"],
            sc["H"], cam.tanfovx, cam.tanfovy)


def vjp64(sc, up, keep, guard, colour_clamped, conic_dropped, variant=None, inputs=None, project_kw=None):
    """The float64 VJP of the upstream `up` through dense64.project, the float32 side's decisions held fixed.
    `inputs`: {name: float64 leaf} (default: the scene's activated inputs); project_kw: project()'s input keywords
    built from them (default: the plain route's).  Returns {name: (P, ...) float64 numpy gradient}."""
    from oracle import dense64

    if inputs is None:
        names = [k for k in PLAIN_INPUTS if k in sc and not (k == "shs" and "colors_precomp" in sc)
                 and not (k in ("scales", "rotations") and "cov3D_precomp" in sc)]
        inputs = {k: sc[k].double().clone().requires_grad_(True) for k in names}
        project_kw = {k: v for k, v in inputs.items() if k not in ("means3D", "opacities")}
        means, opac = inputs["means3D"], inputs["opacities"]
    else:
        means, opac = project_kw.pop("means3D"), project_kw.pop("opacities")
    keep_t = torch.as_tensor(np.asarray(keep, bool))
    pr = dense64.project(means, *cam_args(sc), sh_degree=sc["sh_degree"], scale_modifier=sc["scale_modifier"],
                         guard_clamped=torch.as_tensor(np.asarray(guard, bool)),
                         colour_clamped=None if colour_clamped is None else torch.as_tensor(np.asarray(colour_clamped) != 0),
                         keep=keep_t, conic_dropped=torch.as_tensor(np.asarray(conic_dropped, bool)), variant=variant,
                         **project_kw)
    u = torch.as_tensor(np.asarray(up, np.float64)) * keep_t[:, None]
    conic_up = torch.stack((u[:, 2], 2.0 * u[:, 3], u[:, 4]), 1)   # the off-diagonal entry counts twice
    L = ((u[:, 0:2] * pr["ndc"]).sum() + (conic_up * pr["conic"]).sum() + (u[:, 6:9] * pr["rgb"]).sum()
         + (u[:, 9] * pr["depth"]).sum() + (u[:, 5:6] * opac.reshape(-1, 1)).sum())
    leaves = list(inputs.values())
    grads = torch.autograd.grad(L, leaves, allow_unused=True)
    return {k: (np.zeros(tuple(v.shape)) if gr is None else gr.numpy()) for (k, v), gr in zip(inputs.items(), grads)}


def oracle_vjp(sc, st, up, radii=None, clamped=None):
    """The C oracle's stage 5 fed the same upstream, as float32 numpy: the activated inputs' gradients.  Opacity and
    colors_precomp take their upstream straight through; dL/dz, which the oracle has no slot for, is added to dL/dmeans3D
    in float32 through the view matrix's third column, as the kernels add it."""
    from oracle import rasterizer as orc

    cam = sc["cam"]
    radii = st.radii if radii is None else radii
    vis = (np.asarray(radii) > 0)[:, None]
    kw = oracle_kwargs(sc)
    kw.pop("colors_precomp", None)
    kw.pop("cov3D_precomp", None)
    g = orc.preprocess_backward(st, up[:, 0:2], up[:, 2:5], up[:, 6:9] * vis, sc["means3D"].numpy(),
                                cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
                                cam.camera_center.numpy(), cam.tanfovx, cam.tanfovy, radii=radii, clamped=clamped, **kw)
    V = cam.world_view_transform.numpy().reshape(16).astype(F32)
    gz = (up[:, 9:10] * vis).astype(F32)
    g["means3D"] = g["means3D"] + np.where(vis, gz * V[[2, 6, 10]][None, :], F32(0))
    g["opacities"] = (up[:, 5:6] * vis).astype(F32)
    g["colors_precomp"] = (up[:, 6:9] * vis).astype(F32)
    return g


# The per-splat gate: for every splat row i of a gradient tensor,
#     |dev_i - f64_i|_inf <= 2 |ora_i - f64_i|_inf + (FLOOR + [ill] 4 kappa_i 2^-24) |f64_i|_inf + TINY,
# dev the kernel's float32 gradient, ora the float32 oracle's and f64 the float64 VJP of the same upstream.  Twice the
# oracle's own error leaves room for a different association of the same float32 sums; FLOOR for the rounding of a
# row whose oracle error happens to be smaller; 4 kappa_i 2^-24 (ill_kappa_of) for the splats of adversarial_scenes'
# KNIFE_COND class, whose float32 rounding the covariance chain amplifies about kappa times, a few roundings over
# (a face-on needle of kappa 1e4 was measured at 1.5 kappa 2^-24 in dL/drotations on the CPU oracle).
FLOOR = 2.0 ** -13
# float32's smallest normal: a gradient below it is subnormal noise with no relative precision left (a bound splat's
# dL/d_rotation of 1e-43 against a float64 1e-52 was seen on the H100)
TINY = 2.0 ** -126


def kappa(cov3D):
    c = np.asarray(cov3D, np.float64)
    S = np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], 1)
    ev = np.abs(np.linalg.eigvalsh(S))
    with np.errstate(all="ignore"):
        return np.where(ev[:, 0] > 0, ev[:, 2] / ev[:, 0], np.inf)


def gate_ratio(dev, ora, f64, ill_kappa, floor=FLOOR):
    """(P,) per-splat ratio of |dev_i - f64_i|_inf to its allowance (<= 1 passes; 0 where both sides are exactly
    equal).  ill_kappa: (P,) kappa of the KNIFE_COND splats, 0 elsewhere."""
    P = f64.shape[0]
    d, o, r = (np.asarray(a, np.float64).reshape(P, -1) for a in (dev, ora, f64))
    err = np.abs(d - r).max(1)
    allow = 2.0 * np.abs(o - r).max(1) + (floor + 4.0 * ill_kappa * 2.0 ** -24) * np.abs(r).max(1) + TINY
    with np.errstate(all="ignore"):
        ratio = np.where(err == 0, 0.0, err / allow)
    return np.where(np.isnan(ratio), np.inf, ratio)


def assert_gate(name, dev, ora, f64, ill_kappa, family, what="", floor=FLOOR):
    """Asserts the per-splat gate for one tensor; returns the ratios.  The message names the splat, its family and
    the three values of its row."""
    ratio = gate_ratio(dev, ora, f64, ill_kappa, floor)
    bad = np.nonzero(~(ratio <= 1.0))[0]
    if bad.size:
        i = int(bad[np.argmax(np.where(np.isfinite(ratio[bad]), ratio[bad], np.inf))])
        P = f64.shape[0]
        row = lambda a: np.array2string(np.asarray(a, np.float64).reshape(P, -1)[i], precision=8, max_line_width=400)  # noqa: E731
        raise AssertionError(f"{what} dL/d{name}: {bad.size}/{P} splats beyond the per-splat gate; worst splat {i} "
                             f"({family[i]}, kappa {kappa_note(ill_kappa[i])}) ratio {ratio[i]:.3e}\n"
                             f"  device  {row(dev)}\n  oracle  {row(ora)}\n  float64 {row(f64)}")
    return ratio


def kappa_note(k):
    return f"{k:.2e} (KNIFE_COND)" if k > 0 else "below KNIFE_COND"


def ill_kappa_of(st, pr):
    """(P,) kappa of the KNIFE_COND splats of an oracle state, 0 for every other rendered splat.  The chain amplifies
    float32 rounding by the 3D covariance's condition number and again where det = a c - b^2 of the 2-D covariance
    cancels, by cond2 = (|a c| + b^2) / |det| (pr: f32_project of the state): kappa is the larger of the two, and a
    splat is of the class when either is beyond KNIFE_COND."""
    a, b, c = pr["cov2d"].astype(np.float64).T
    with np.errstate(all="ignore"):
        cond2 = (np.abs(a * c) + b * b) / np.abs(pr["det"].astype(np.float64))
    k = np.fmax(kappa(st.cov3D), cond2)
    return np.where((st.radii > 0) & (k > A.KNIFE_COND), k, 0.0)


def percentiles(ratio):
    r = np.sort(ratio[np.isfinite(ratio)])
    q = lambda f: float(r[min(len(r) - 1, int(f * len(r)))]) if len(r) else 0.0  # noqa: E731
    return q(0.5), q(0.99), float(r[-1]) if len(r) else 0.0
