"""Shared scene builders / comparison helpers for the tests (CPU oracle on one side, CUDA path on the other)."""
from __future__ import annotations

import numpy as np
import torch

from gaussianavatars_b200 import synthetic as syn
from oracle import binding as ob
from oracle import rasterizer as orc

# Parity budget (north_star): <= 1e-4 max abs per channel.  Two independent implementations of
#   alpha = min(.99, o * exp(power));  skip if alpha < 1/255;  stop if T(1-alpha) < 1e-4
# disagree on those THRESHOLD DECISIONS at knife edges (exp differs by ~1 ulp), which moves an isolated pixel by up
# to ~alpha*T*c <= 1/255.  So: every pixel within KNIFE_ABS, and all but a KNIFE_FRAC fraction within 1e-4.
IMG_TOL = 1e-4
KNIFE_ABS = 1.2e-2
KNIFE_FRAC = 2e-5


def assert_image_close(img_cuda: np.ndarray, img_ref: np.ndarray, what="", frac=KNIFE_FRAC):
    d = np.abs(img_cuda.astype(np.float64) - img_ref.astype(np.float64))
    n_bad = int((d > IMG_TOL).sum())
    assert d.max() <= KNIFE_ABS, f"{what}: max abs diff {d.max():.3e} beyond even a threshold flip"
    assert n_bad <= max(2, frac * d.size), f"{what}: {n_bad}/{d.size} values differ by more than {IMG_TOL}"
    return d.max(), n_bad


def assert_grad_close(g_cuda: np.ndarray, g_ref: np.ndarray, what="", rtol=2e-3, frac=1e-3):
    """Gradient parity is tolerance-based by construction (the reference accumulates with float atomics in
    nondeterministic order, Appendix B.4).  Scale: the largest reference magnitude of that tensor."""
    g_cuda = g_cuda.astype(np.float64).reshape(g_ref.shape)
    g_ref = g_ref.astype(np.float64)
    assert np.isfinite(g_cuda).all(), f"{what}: non-finite gradient"
    scale = np.abs(g_ref).max() + 1e-30
    err = np.abs(g_cuda - g_ref) / scale
    n_bad = int((err > rtol).sum())
    assert n_bad <= max(3, frac * err.size), f"{what}: {n_bad}/{err.size} entries off by > {rtol} of max|ref| (worst {err.max():.3e})"
    return err.max(), n_bad


# Bounded elementwise gradient gate (used by the full-size parity tests; VERDICT r01 "tighten the gradient gate"):
#   |d| <= atol + rtol |ref|  for every entry, with atol a fixed fraction of the tensor's largest reference magnitude
#   (float accumulation-order noise of sums with cancellation scales with the terms, not with the result);
#   the few entries beyond it (threshold knife edges: one (pixel, splat) pair accepted on one side and skipped on the
#   other) are counted, must stay below `max_outlier_frac`, and none may exceed `cap` x max|ref|.
GRAD_RTOL = 1e-3
GRAD_ATOL_FRAC = 2e-5
GRAD_OUTLIER_FRAC = 1e-4
GRAD_CAP = 1e-2


def grad_stats(g_cuda: np.ndarray, g_ref: np.ndarray, rtol=GRAD_RTOL, atol_frac=GRAD_ATOL_FRAC):
    g_ref = np.asarray(g_ref, np.float64)
    g_cuda = np.asarray(g_cuda, np.float64).reshape(g_ref.shape)
    scale = float(np.abs(g_ref).max()) + 1e-300
    d = np.abs(g_cuda - g_ref)
    tol = atol_frac * scale + rtol * np.abs(g_ref)
    ratio = d / tol
    flat = np.sort(ratio.reshape(-1))
    q = lambda f: float(flat[min(len(flat) - 1, int(f * len(flat)))]) if len(flat) else 0.0  # noqa: E731
    return dict(n=int(d.size), finite=bool(np.isfinite(g_cuda).all()), scale=scale, max_abs_over_scale=float(d.max() / scale) if d.size else 0.0,
                p50=q(0.5), p999=q(0.999), worst=float(flat[-1]) if len(flat) else 0.0, outliers=int((ratio > 1.0).sum()))


def assert_grad_tight(g_cuda, g_ref, what="", rtol=GRAD_RTOL, atol_frac=GRAD_ATOL_FRAC,
                      max_outlier_frac=GRAD_OUTLIER_FRAC, cap=GRAD_CAP, min_outliers_allowed=8):
    s = grad_stats(g_cuda, g_ref, rtol, atol_frac)
    print(f"[grad] {what:<28s} n={s['n']:>9d} max|ref|={s['scale']:.3e} worst|d|/max|ref|={s['max_abs_over_scale']:.2e} "
          f"tol-ratio p50={s['p50']:.2e} p99.9={s['p999']:.2e} worst={s['worst']:.2e} outliers={s['outliers']}")
    assert s["finite"], f"{what}: non-finite gradient"
    assert s["max_abs_over_scale"] <= cap, f"{what}: worst entry off by {s['max_abs_over_scale']:.3e} of max|ref| (cap {cap})"
    allowed = max(min_outliers_allowed, int(max_outlier_frac * s["n"]))
    assert s["outliers"] <= allowed, (f"{what}: {s['outliers']}/{s['n']} entries beyond atol+rtol|ref| "
                                      f"(rtol {rtol}, atol {atol_frac} max|ref|; allowed {allowed})")
    return s


# Explained gates: the outliers the gates above let through by count must each sit where a threshold decision can
# flip (tests/adversarial_scenes.py::knife_edges).  Every entry outside that set is within the tolerance, without
# exception; the entries inside it keep the cap.
def _affected(mask, shape):
    mask = np.asarray(mask, bool)
    return np.broadcast_to(mask.reshape(mask.shape + (1,) * (len(shape) - mask.ndim)), shape)


def assert_grad_explained(g_cuda, g_ref, affected, what="", rtol=GRAD_RTOL, atol_frac=GRAD_ATOL_FRAC, cap=GRAD_CAP,
                          knife_allowed=None):
    """`affected`: boolean mask of the entries a knife edge explains, of the tensor's shape or of its leading
    dimensions (the (P,) splat mask of knife_edges).  The affected entries keep assert_grad_tight's allowance: at
    most `knife_allowed` (default max(8, GRAD_OUTLIER_FRAC n)) beyond the tolerance, none beyond `cap` max|ref|."""
    g_ref = np.asarray(g_ref, np.float64)
    g_cuda = np.asarray(g_cuda, np.float64).reshape(g_ref.shape)
    aff = _affected(affected, g_ref.shape)
    scale = float(np.abs(g_ref).max()) + 1e-300 if g_ref.size else 1.0
    d = np.abs(g_cuda - g_ref)
    ratio = d / (atol_frac * scale + rtol * np.abs(g_ref))
    free = ratio[~aff]
    worst_free = float(free.max()) if free.size else 0.0
    worst_knife = float(d[aff].max() / scale) if aff.any() else 0.0
    n_bad = int((free > 1.0).sum())
    print(f"[grad] {what:<28s} n={d.size:>9d} max|ref|={scale:.3e} knife={int(aff.sum())} "
          f"tol-ratio worst={worst_free:.2e} outside the knife set, knife worst|d|/max|ref|={worst_knife:.2e} "
          f"unexplained={n_bad}")
    assert np.isfinite(g_cuda).all(), f"{what}: non-finite gradient"
    if n_bad:
        at = np.unravel_index(int(np.argmax(np.where(aff, -1.0, ratio))), ratio.shape)
        raise AssertionError(f"{what}: {n_bad}/{d.size} entries outside the knife set beyond atol+rtol|ref| (rtol {rtol}, "
                             f"atol {atol_frac} max|ref|); worst ratio {worst_free:.3e} at {tuple(map(int, at))}: "
                             f"{g_cuda[at]:.6e} vs {g_ref[at]:.6e}")
    assert worst_knife <= cap, f"{what}: a knife entry off by {worst_knife:.3e} of max|ref| (cap {cap})"
    allowed = max(8, int(GRAD_OUTLIER_FRAC * d.size)) if knife_allowed is None else knife_allowed
    n_knife = int((ratio[aff] > 1.0).sum())
    assert n_knife <= allowed, f"{what}: {n_knife} knife entries beyond atol+rtol|ref| (allowed {allowed})"
    return dict(n=int(d.size), knife=int(aff.sum()), worst=worst_free, knife_worst=worst_knife)


def assert_image_explained(img_cuda, img_ref, knife_pixels, what="", tol=IMG_TOL, cap=KNIFE_ABS, frac=KNIFE_FRAC):
    """Every value of a pixel outside `knife_pixels` ((H, W), broadcast over leading channels) within `tol`; the knife
    pixels keep assert_image_close's allowance: at most max(2, frac n) values beyond `tol`, none beyond `cap`."""
    img_ref = np.asarray(img_ref, np.float64)
    d = np.abs(np.asarray(img_cuda, np.float64).reshape(img_ref.shape) - img_ref)
    kp = np.asarray(knife_pixels, bool)
    aff = np.broadcast_to(kp.reshape((1,) * (d.ndim - kp.ndim) + kp.shape), d.shape)
    free = d[~aff]
    worst_free = float(free.max()) if free.size else 0.0
    worst_knife = float(d[aff].max()) if aff.any() else 0.0
    n_bad = int((free > tol).sum())
    print(f"[image] {what:<28s} n={d.size:>9d} knife pixels={int(kp.sum())} max|d| outside={worst_free:.3e} "
          f"knife max|d|={worst_knife:.3e} unexplained={n_bad}")
    if n_bad:
        at = np.unravel_index(int(np.argmax(np.where(aff, -1.0, d))), d.shape)
        raise AssertionError(f"{what}: {n_bad}/{d.size} values outside the knife pixels differ by more than {tol}; "
                             f"worst {worst_free:.3e} at {tuple(map(int, at))}")
    assert worst_knife <= cap, f"{what}: a knife pixel off by {worst_knife:.3e} (cap {cap})"
    n_knife = int((d[aff] > tol).sum())
    assert n_knife <= max(2, frac * d.size), f"{what}: {n_knife} knife-pixel values differ by more than {tol}"
    return worst_free, worst_knife


def image_stats(img_cuda: np.ndarray, img_ref: np.ndarray):
    d = np.abs(img_cuda.astype(np.float64) - img_ref.astype(np.float64))
    return dict(max_abs=float(d.max()), n_over_1e4=int((d > IMG_TOL).sum()), n=int(d.size))


def carve(sizes):
    """Byte offsets of consecutive Carver::take calls (256-B aligned), as csrc/common.cuh lays the buffers out."""
    off, out = 0, []
    for s in sizes:
        off = (off + 255) & ~255
        out.append(off)
        off += s
    return out


def buffer(holder, ptr):
    """The tensor of a frame's scratch holder that starts at device address `ptr`."""
    return next(t for t in holder if t.data_ptr() == ptr)


def random_scene(P=10_000, W=256, H=256, sh_degree=0, seed=0, fov=60.0, scale_shift=0.0, max_sh_degree=None):
    """Config-1 style scene: activated (reference-surface) inputs as CPU float32 tensors."""
    sp = syn.random_splats(P, seed=seed, sh_degree=sh_degree, max_sh_degree=max_sh_degree)
    cam = syn.look_at_camera(W, H, fov, fov * H / W if H != W else fov)
    scene = dict(
        means3D=sp["_xyz"].contiguous(),
        scales=ob.get_scaling(sp["_scaling"] + scale_shift).contiguous(),
        rotations=ob.get_rotation(sp["_rotation"]).contiguous(),
        opacities=ob.get_opacity(sp["_opacity"]).contiguous(),
        shs=ob.get_features(sp["_features_dc"], sp["_features_rest"]).contiguous(),
        raw=sp, cam=cam, W=W, H=H, sh_degree=sh_degree, bg=torch.tensor([0.1, 0.4, 0.8]))
    return scene


def oracle_forward(scene, **over):
    cam = scene["cam"]
    kw = dict(shs=scene["shs"].numpy(), sh_degree=scene["sh_degree"], scales=scene["scales"].numpy(),
              rotations=scene["rotations"].numpy())
    kw.update(over)
    return orc.forward(scene["means3D"].numpy(), scene["opacities"].numpy(), cam.world_view_transform.numpy(),
                       cam.full_proj_transform.numpy(), cam.camera_center.numpy(), scene["W"], scene["H"],
                       cam.tanfovx, cam.tanfovy, scene["bg"].numpy(), **kw)


def oracle_backward(scene, st, dL_dpix, **over):
    cam = scene["cam"]
    kw = dict(shs=scene["shs"].numpy(), sh_degree=scene["sh_degree"], scales=scene["scales"].numpy(),
              rotations=scene["rotations"].numpy())
    kw.update(over)
    return orc.backward(st, dL_dpix, scene["means3D"].numpy(), cam.world_view_transform.numpy(),
                        cam.full_proj_transform.numpy(), cam.camera_center.numpy(), cam.tanfovx, cam.tanfovy,
                        scene["bg"].numpy(), **kw)


def cuda_settings(scene, device, debug=True, scale_modifier=1.0):
    from gaussianavatars_b200 import GaussianRasterizationSettings

    cam = scene["cam"]
    return GaussianRasterizationSettings(
        image_height=scene["H"], image_width=scene["W"], tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
        bg=scene["bg"].to(device), scale_modifier=scale_modifier, viewmatrix=cam.world_view_transform.to(device),
        projmatrix=cam.full_proj_transform.to(device), sh_degree=scene["sh_degree"],
        campos=cam.camera_center.to(device), prefiltered=False, debug=debug)


def avatar_scene(P=20_000, W=480, H=352, seed=0, timestep=2, n_lat=26, n_lon=48, sh_degree=3, scale_gain=2.5,
                 azimuth=15.0):
    """Bound (fused-surface) scene: raw parameters + mesh; the oracle side evaluates the eager getters on CPU."""
    verts, faces = syn.head_mesh(n_lat=n_lat, n_lon=n_lon, seed=seed)
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=seed, sh_degree=sh_degree, scale_gain=scale_gain)
    cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=azimuth)
    v = syn.pose_mesh(verts, timestep)
    return dict(params=params, verts=v, faces=faces, cam=cam, W=W, H=H, sh_degree=sh_degree,
                bg=torch.tensor([1.0, 1.0, 1.0]))


def avatar_activated(sc, dtype=torch.float32, requires_grad=False):
    """Eager reference route on CPU (autograd-capable): returns dict of activated tensors + the leaf tensors."""
    p = sc["params"]
    leaves = {k: p[k].to(dtype).clone().requires_grad_(requires_grad)
              for k in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")}
    verts = sc["verts"].to(dtype).clone().requires_grad_(requires_grad)
    b = p["binding"].long()
    fr = ob.update_mesh_properties(verts, sc["faces"])
    act = dict(
        means3D=ob.get_xyz(leaves["_xyz"], b, fr["face_center"], fr["face_orien_mat"], fr["face_scaling"]),
        scales=ob.get_scaling(leaves["_scaling"], b, fr["face_scaling"]),
        rotations=ob.get_rotation(leaves["_rotation"], b, fr["face_orien_quat"]),
        opacities=ob.get_opacity(leaves["_opacity"]),
        shs=ob.get_features(leaves["_features_dc"], leaves["_features_rest"]))
    return act, leaves, verts, fr
