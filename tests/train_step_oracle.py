"""One mesh-bound training step of the reference, composed from the test oracles, and the gates a CUDA step is held to.

TEST INFRASTRUCTURE.  The step is the chain that trains a GaussianAvatars head (train.py:118-150):

    select_mesh_by_timestep      FLAME forward of row t               tests/flame_oracle.py
    update_mesh_properties       face centre, frame and scale          oracle/binding.py
    getters                      get_xyz / get_scaling / get_rotation (quaternion detour) / get_opacity / get_features
    render                       float64: oracle/dense64.py; float32: the C oracle (oracle/rasterizer.py)
    photometric loss             oracle/loss.py::photometric_torch, lambda_dssim 0.2
    xyz / scale regularisers     train.py:134-146 as written, visibility = radii > 0 of this render
    total.backward()

and `step()` returns what every link of it hands back: the loss parts, the six raw splat gradients, dL/dmeans2D,
dL/dverts, the six posed FLAME gradients and the radii.

Two arithmetics:
  * float64, the yardstick.  The render's discrete decisions -- radii, the tile rectangles' centres and the depth
    order -- are pinned (`pin`) to the float32 C oracle evaluated on a given float32 activation, so that both sides
    blend the same splats in the same order; everything continuous is float64 autograd.
  * float32, the reference's own order of operations: the same chain with the C oracle's autograd as the render.  It
    is what the reference itself computes, and what shows that a gate is not stricter than the reference: a gate
    that the float32 chain fails is wrong, not the kernel.

`mutation=` switches on one deliberately wrong variant of the float64 chain (MUTATIONS); a gate that does not reject
each of them on the scene it checks cannot see the bug that mutation stands for.
"""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import binding as ob
from oracle import dense64
from oracle import rasterizer as orc
from oracle.fused_reference import RAW
from oracle.loss import photometric_torch
from tests import flame_oracle as fo
from tests import helpers as h

LOSS_PARTS = ("l1", "ssim", "xyz", "scale", "total")
REG_KEYS = ("threshold_xyz", "threshold_scale", "lambda_xyz", "lambda_scale", "metric_xyz", "metric_scale")
MUTATIONS = {
    "a": "R^T x in place of R x in get_xyz",
    "b": "face_scaling detached inside get_xyz",
    "c": "metric regularisers computed non-metric (their face_scaling term dropped)",
    "d": "each face-centre gradient sent entirely to the face's first vertex",
    "e": "the means2D x / y pixel scales swapped",
    "f": "dL/dface_scaling scaled by 1.01",
}
CSR_CHUNK = 16   # splats per chunk of the backward's per-face reduction (rasterizer._face_csr)


def flags(sh_degree=3, metric=False, **over):
    """The frame's settings: active SH degree, background, lambda_dssim and the regulariser arguments of
    train.py:134-146 (arguments/__init__.py:100-105 defaults; `metric` switches both metric_* flags)."""
    f = dict(sh_degree=sh_degree, bg=(1.0, 1.0, 1.0), lambda_dssim=0.2, threshold_xyz=1.0, threshold_scale=0.6,
             lambda_xyz=1e-2, lambda_scale=1.0, metric_xyz=metric, metric_scale=metric)
    f.update(over)
    return f


def reg_kwargs(fl):
    return {k: fl[k] for k in REG_KEYS}


def pin_of(st):
    """The discrete decisions of a float32 C-oracle forward that the float64 render takes over."""
    return dict(radii=np.asarray(st.radii).copy(), xy=np.asarray(st.xy).copy(), depths=np.asarray(st.depths).copy())


def oracle_forward_on(means3D, opacities, cam, W, H, fl, shs, scales=None, rotations=None, cov3D=None):
    """The float32 C oracle's forward on a given float32 activation (the CUDA path's exported one, say)."""
    n = lambda t: None if t is None else t.detach().float().cpu().contiguous().numpy()   # noqa: E731
    return orc.forward(n(means3D), n(opacities), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
                       cam.camera_center.numpy(), W, H, cam.tanfovx, cam.tanfovy, np.asarray(fl["bg"], np.float32),
                       shs=n(shs), sh_degree=fl["sh_degree"], scales=n(scales), rotations=n(rotations),
                       cov3D_precomp=n(cov3D))


def _render32(act, cam, W, H, fl, P):
    RS = namedtuple("RS", "image_height image_width tanfovx tanfovy bg scale_modifier viewmatrix projmatrix sh_degree "
                          "campos prefiltered debug")
    rs = RS(H, W, cam.tanfovx, cam.tanfovy, torch.tensor(fl["bg"], dtype=torch.float32), 1.0,
            cam.world_view_transform, cam.full_proj_transform, fl["sh_degree"], cam.camera_center, False, False)
    Fn = orc.make_autograd_function()
    holder = {}

    class Keep(Fn):
        @staticmethod
        def forward(ctx, *a):
            out = Fn.forward(ctx, *a)
            holder["st"] = ctx.st
            return out

        @staticmethod
        def backward(ctx, *g):
            return Fn.backward(ctx, *g)

    m2 = torch.zeros(P, 3, requires_grad=True)
    img, radii = Keep.apply(act["means3D"], m2, act["shs"].contiguous(), None, act["opacities"], act["scales"],
                            act["rotations"], None, rs)
    return img, radii.long(), m2, holder["st"]


def _render64(act, cam, W, H, fl, P, pin, mutation):
    radii = torch.from_numpy(pin["radii"]).long()
    idx = torch.nonzero(radii > 0).reshape(-1)   # splats without a radius reach no pixel: leave them out of the
    d = torch.float64                            # (H W, P) tensors
    m2 = torch.zeros(P, 3, dtype=d, requires_grad=True)
    m2_used = m2
    if mutation == "e":   # value unchanged (zero), gradient scaled by H/W on x and W/H on y
        m2_used = m2 * torch.tensor([H / W, W / H, 1.0], dtype=d)
    img, aux = dense64.render(act["means3D"][idx], m2_used[idx], act["opacities"][idx], cam.world_view_transform.to(d),
                              cam.full_proj_transform.to(d), cam.camera_center.to(d), W, H, cam.tanfovx, cam.tanfovy,
                              torch.tensor(fl["bg"], dtype=d), shs=act["shs"][idx], sh_degree=fl["sh_degree"],
                              scales=act["scales"][idx], rotations=act["rotations"][idx], radii=radii[idx],
                              rect_xy=torch.from_numpy(pin["xy"])[idx], depths=torch.from_numpy(pin["depths"])[idx])
    return img, radii, m2, aux


def regularizers(_xyz, _scaling, scales, fs_b, vis, fl, mutation=None):
    """losses['xyz'], losses['scale'] of train.py:134-146, with get_scaling = `scales` (the render's own tensor)."""
    metric_xyz = fl["metric_xyz"] and mutation != "c"
    metric_scale = fl["metric_scale"] and mutation != "c"
    if metric_xyz:
        lx = F.relu((_xyz * fs_b)[vis] - fl["threshold_xyz"]).norm(dim=1).mean() * fl["lambda_xyz"]
    else:
        lx = F.relu(_xyz[vis].norm(dim=1) - fl["threshold_xyz"]).mean() * fl["lambda_xyz"]
    ls = _xyz.new_zeros(())
    if fl["lambda_scale"] != 0:
        if metric_scale:
            ls = F.relu(scales[vis] - fl["threshold_scale"]).norm(dim=1).mean() * fl["lambda_scale"]
        else:
            ls = F.relu(torch.exp(_scaling[vis]) - fl["threshold_scale"]).norm(dim=1).mean() * fl["lambda_scale"]
    return lx, ls


def reg_active(_xyz, _scaling, scales, fs_b, fl):
    """Per splat: does each regulariser term have a non-zero value (before the visibility filter)?"""
    if fl["metric_xyz"]:
        ax = ((_xyz * fs_b) > fl["threshold_xyz"]).any(dim=1)
    else:
        ax = _xyz.norm(dim=1) > fl["threshold_xyz"]
    s = scales if fl["metric_scale"] else torch.exp(_scaling)
    return ax, (s > fl["threshold_scale"]).any(dim=1)


def step(params, flame_param, t, assets, cam, gt_u8, fl, dtype, pin=None, mutation=None):
    """One training step of the reference on the CPU in `dtype` (float64 needs `pin`, see the module docstring).

    params: raw splat parameters + int `binding`; flame_param: the reference's per-timestep dict; assets: FLAME assets
    with `faces`; cam: a synthetic camera; gt_u8: (3, H, W) uint8; fl: flags().  Returns a dict: parts {LOSS_PARTS:
    float}, grads {raw name: array, 'means2D', 'verts'}, flame {posed name: (T, n) array}, radii, and the state the
    regime checks read (float32: the oracle state `st` and its `pin`; float64: the dense model's `aux`)."""
    if mutation is not None and (dtype != torch.float64 or mutation not in MUTATIONS):
        raise ValueError("mutations apply to the float64 chain: one of " + ", ".join(MUTATIONS))
    if dtype == torch.float64 and pin is None:
        raise ValueError("the float64 render needs the pinned decisions of a float32 oracle forward (pin=)")
    H, W = int(gt_u8.shape[1]), int(gt_u8.shape[2])
    a = fo.assets_as({k: assets[k] for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights",
                                             "parents")}, dtype)
    fp = {k: v.to(dtype).clone() for k, v in flame_param.items() if v is not None and k != "dynamic_offset"}
    for k in fo.POSED:
        fp[k].requires_grad_(True)
    verts = fo.select_mesh_by_timestep(a, fp, t)[0][0]
    verts.retain_grad()
    faces = assets["faces"].long()
    leaves = {k: params[k].to(dtype).clone().requires_grad_(True) for k in RAW}
    b = params["binding"].long()
    P = b.shape[0]

    fr = ob.update_mesh_properties(verts, faces)
    fc, fR, fs = fr["face_center"], fr["face_orien_mat"], fr["face_scaling"]
    if mutation == "d":
        v0, v1, v2 = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
        fc = v0 + ((v1 + v2 - 2 * v0) / 3).detach()
    if mutation == "f":
        fs = fs * 1.01 - (0.01 * fs).detach()
    act = dict(
        means3D=ob.get_xyz(leaves["_xyz"], b, fc, fR.transpose(-1, -2) if mutation == "a" else fR,
                           fs.detach() if mutation == "b" else fs),
        scales=ob.get_scaling(leaves["_scaling"], b, fs),
        rotations=ob.get_rotation(leaves["_rotation"], b, fr["face_orien_quat"]),
        opacities=ob.get_opacity(leaves["_opacity"]),
        shs=ob.get_features(leaves["_features_dc"], leaves["_features_rest"]))

    out = {}
    if dtype == torch.float64:
        img, radii, m2, aux = _render64(act, cam, W, H, fl, P, pin, mutation)
        out["aux"] = {k: v.detach() if isinstance(v, torch.Tensor) else v for k, v in aux.items()}
    else:
        img, radii, m2, st = _render32(act, cam, W, H, fl, P)
        out["st"], out["pin"] = st, pin_of(st)
    gt = gt_u8.to(dtype) / 255.0
    l1, ssim, photo = photometric_torch(img, gt, fl["lambda_dssim"])
    vis = radii > 0
    lx, ls = regularizers(leaves["_xyz"], leaves["_scaling"], act["scales"], fs[b], vis, fl, mutation)
    total = photo + lx + ls
    total.backward()

    n = lambda x: x.detach().numpy()   # noqa: E731
    out.update(image=n(img), radii=radii.numpy(), vis=vis.numpy(),
               parts={k: float(v.detach()) for k, v in zip(LOSS_PARTS, (l1, ssim, lx, ls, total))},
               grads={**{k: n(leaves[k].grad) for k in RAW}, "means2D": n(m2.grad), "verts": n(verts.grad)},
               flame={k: n(fp[k].grad) for k in fo.POSED},
               reg_active=[n(x) for x in reg_active(leaves["_xyz"], leaves["_scaling"], act["scales"], fs[b], fl)],
               activation={k: n(v) for k, v in act.items()}, l1_sign=n(torch.sign(img - gt)))
    return out


# ---- gates ------------------------------------------------------------------------------------------------------------
# Fixed before any CUDA number was seen.  Per-splat arrays: helpers.assert_grad_tight at its defaults (the gate the
# unbound adversarial suite passes).  Per-vertex and FLAME arrays: |d| <= 1e-3 |ref64| + 1e-4 max|ref64| elementwise,
# at most max(8, 1e-4 n) entries beyond it -- and never more than n / 8, so that a FLAME row of 3 or 6 entries is not
# waved through by the allowance -- none beyond 1e-2 max|ref64|.  Loss parts: 2e-6 absolute; the regularisers also
# 2e-6 relative.
SPLAT_KEYS = RAW + ("means2D",)
LOSS_ABS, REG_REL = 2e-6, 2e-6
VERT_RTOL, VERT_ATOL = 1e-3, 1e-4


def _grad_gate(what, got, ref, rtol, atol_frac, small_cap):
    s = h.grad_stats(got, ref, rtol=rtol, atol_frac=atol_frac)
    allowed = max(8, int(h.GRAD_OUTLIER_FRAC * s["n"]))
    if small_cap:
        allowed = min(allowed, s["n"] // 8)
    s.update(what=what, allowed=allowed,
             ok=bool(s["finite"] and s["max_abs_over_scale"] <= h.GRAD_CAP and s["outliers"] <= allowed))
    return s


def gate_splat(what, got, ref):
    return _grad_gate(what, got, ref, h.GRAD_RTOL, h.GRAD_ATOL_FRAC, small_cap=False)


def gate_vertex(what, got, ref):
    return _grad_gate(what, got, ref, VERT_RTOL, VERT_ATOL, small_cap=True)


def gate_loss(what, got, ref):
    d = abs(float(got) - float(ref))
    tol = LOSS_ABS
    ok = d <= LOSS_ABS
    if what in ("xyz", "scale"):
        ok = ok and d <= REG_REL * abs(float(ref))
        tol = min(LOSS_ABS, REG_REL * abs(float(ref))) if ref != 0 else 0.0
    ratio = d / tol if tol > 0 else (0.0 if d == 0 else float("inf"))
    return dict(what=what, n=1, worst=ratio, p50=ratio, p999=ratio, outliers=int(not ok), allowed=0, ok=bool(ok),
                max_abs_over_scale=d)


def gates(got, ref, t, keys=None):
    """Every gate of one step against the float64 step `ref`.  `got` holds what a route produced, in step()'s layout
    (missing entries are skipped: a graph replay has no dL/dverts).  Returns a list of gate records."""
    res = []
    for k in LOSS_PARTS:
        if k in got.get("parts", {}):
            res.append(gate_loss(k, got["parts"][k], ref["parts"][k]))
    for k in SPLAT_KEYS:
        if k in got.get("grads", {}):
            res.append(gate_splat(f"dL/d{k}", got["grads"][k], ref["grads"][k]))
    if "xyz_gradient_accum" in got:
        acc = np.linalg.norm(ref["grads"]["means2D"][:, :2].astype(np.float64), axis=1)[:, None]
        res.append(gate_splat("xyz_gradient_accum", got["xyz_gradient_accum"], acc))
    if "verts" in got.get("grads", {}):
        res.append(gate_vertex("dL/dverts", got["grads"]["verts"], ref["grads"]["verts"]))
    for k in fo.POSED:
        if k in got.get("flame", {}):
            g = np.asarray(got["flame"][k])
            s = gate_vertex(f"dL/d{k}[t]", g[t], ref["flame"][k][t])
            rest = np.delete(g, t, axis=0)
            if np.count_nonzero(rest):
                s["ok"] = False
                s["what"] += " (rows other than t not zero)"
            res.append(s)
    return [r for r in res if keys is None or r["what"] in keys]


def report(title, recs):
    for r in recs:
        print(f"[train-step] {title:<34s} {r['what']:<26s} tol-ratio p50={r['p50']:.2e} p99.9={r['p999']:.2e} "
              f"worst={r['worst']:.2e} outliers={r['outliers']}/{r['allowed']} {'ok' if r['ok'] else 'FAIL'}")


def failed(recs):
    return [r["what"] for r in recs if not r["ok"]]


# ---- scenes -----------------------------------------------------------------------------------------------------------
def flame_sequence(a, T=7, seed=0):
    """A FLAME track over the assets `a`: smooth rows, then (T >= 7) row 4 with neck / jaw / eyes exactly zero and
    row 6 at 2.5 rad per joint (as tests/test_gpu_flame.py's full-size sequence)."""
    from gaussianavatars_b200 import synthetic as syn
    fp = syn.flame_like_sequence(T, seed=seed + 1, V=a["v_template"].shape[0])
    fp.pop("dynamic_offset")
    if T >= 7:
        g = torch.Generator().manual_seed(seed)
        for k in ("neck_pose", "jaw_pose", "eyes_pose"):
            fp[k][4] = 0.0
            d = torch.randn(fp[k].shape[1], generator=g)
            fp[k][6] = 2.5 * d / d.norm() * (fp[k].shape[1] // 3) ** 0.5
        fp["rotation"][6] = torch.tensor([1.5, -1.8, 0.9]) * 2.5 / 2.5495
    return fp


def scene(P=2_500, W=96, H=72, seed=0, scale_shift=0.0, sh_degree=3, azimuth=15.0, hot=(120, 56), far=0.02):
    """FLAME-like head (synthetic.flame_like_assets), its track, P splats with the heavy-tailed binding, the orbit
    camera at W x H and a seeded uint8 ground truth.  On top of synthetic.avatar_splats: `scale_shift` moves the raw
    _scaling; the first splats are moved onto `hot` faces that own that many (a face spanning several chunks of the
    per-face reduction); a `far` fraction of splats sits 60 face scales off its face, off screen (radius 0)."""
    from gaussianavatars_b200 import synthetic as syn
    a = syn.flame_like_assets(seed)
    fp = flame_sequence(a, seed=seed)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=seed + 3, sh_degree=sh_degree, scale_gain=2.5)
    params["_scaling"] = params["_scaling"] + scale_shift
    b, start = params["binding"], 0
    for n in hot:
        b[start:start + n] = b[start]
        start += n
    g = torch.Generator().manual_seed(seed + 5)
    off = torch.rand(P, generator=g) < far
    params["_xyz"][off] *= 60.0
    cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=azimuth)
    gt = torch.randint(0, 256, (3, H, W), generator=torch.Generator().manual_seed(seed + 7), dtype=torch.uint8)
    return dict(params=params, flame_param=fp, assets=a, cam=cam, gt=gt, W=W, H=H)


def metric_flags(sc, sh_degree=3):
    """metric_xyz = metric_scale = True.  The metric terms compare world lengths with the thresholds, so 1 and 0.6
    are taken in units of the median face scale of the rest mesh (a few millimetres on this head): at 1 and 0.6 metres
    neither term would ever be non-zero."""
    v = sc["assets"]["v_template"].double()
    fs = ob.update_mesh_properties(v, sc["assets"]["faces"].long())["face_scaling"]
    m = float(fs.median())
    return flags(sh_degree, metric=True, threshold_xyz=1.0 * m, threshold_scale=0.6 * m)


def run_pair(sc, t, fl, mutation=None):
    """The float32 reference-order step and the float64 step pinned to its oracle forward."""
    args = (sc["params"], sc["flame_param"], t, sc["assets"], sc["cam"], sc["gt"], fl)
    r32 = step(*args, torch.float32)
    r64 = step(*args, torch.float64, pin=r32["pin"])
    return r32, r64


# ---- regimes ----------------------------------------------------------------------------------------------------------
def regimes(params, n_faces, r64, r32):
    """What a scene reaches, from the oracles' own state (see test_oracle_train_step)."""
    b = params["binding"].long()
    counts = torch.bincount(b, minlength=n_faces).numpy()
    chunks = (counts + CSR_CHUNK - 1) // CSR_CHUNK
    aux = r64["aux"]
    covered = aux["n_keep"].numpy() > 0
    vis = r64["vis"]
    ax, asc = r64["reg_active"]
    opac = torch.sigmoid(params["_opacity"].double()).numpy().reshape(-1)
    return dict(max_chunks=int(chunks.max()), empty_face_frac=float((counts == 0).mean()),
                mean_contrib=float(aux["n_keep"].numpy()[covered].mean()) if covered.any() else 0.0,
                low_T_frac=float((aux["T_final"].numpy() < 0.5).mean()),
                xyz_active=float((ax & vis).sum() / max(vis.sum(), 1)),
                scale_active=float((asc & vis).sum() / max(vis.sum(), 1)),
                radius0=int((r64["radii"] == 0).sum()), faint=int(((opac < 1 / 255) & vis).sum()))
