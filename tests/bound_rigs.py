"""Mesh-bound camera rigs at the geometric edges (TEST INFRASTRUCTURE): the adversarial scenes of
tests/adversarial_scenes.py turned into raw parameters on a triangle mesh, seen by several cameras that each put the
same splats at a different edge.

`bind(sc)` inverts the getters of oracle/binding.py for an activated scene: per splat
    _xyz = R_f^T (x - c_f) / fs_f,  _rotation = q_f^-1 (x) q (times a random norm),  _scaling = log(s / fs_f),
    _opacity = logit(o),  _features_dc / _features_rest = the scene's SH rows,
computed in float64 on the float32 mesh and rounded once.  Faces are of two kinds, alternating:
    exact    axis-aligned right triangles with legs 2^k on a 1/1024 grid: R_f is a signed permutation, fs = 2^k
    general  random orientation, fs in [0.5, 2], centre up to 0.3 off the mean of its splats
Face 0 holds more than 64 splats when the scene has enough (several chunks of the per-face reduction), three faces
hold none, and splats are dealt to faces at random, so neighbouring splats sit on different faces.  The rounding
through the binding moves float32 knife edges by an ulp or so: callers compare against the activation the CUDA path
exports (rasterizer.bind_activate), not against the scene.  SH degree 0 scenes get three more stored coefficients, so
every rig also has unused SH coefficients.

`rig(bound, K)` returns the first K of six cameras of the scene's image size:
    0  the builder's camera (identity view, looking down +z)
    1  the same pose at 0.8 x tan(FoV/2): splats with 1.04 < |x/z| / tan < 1.3 are inside view 0's guard band and
       outside this one's
    2  a dolly of DOLLY along +z: the band 0.2 < z <= 0.2 + DOLLY is culled at the near plane here, visible in view 0
    3  the camera turned around behind the scene (180 degrees about y, at z = max z + 1): the depth order reverses and
       equal depths stay equal; splats view 0 culls at the near plane are in front of it
    4  view 0 again
    5  view 0 with tan(FoV/2) = 0: an invalid field of view, every splat culled
"""
from __future__ import annotations

import math

import numpy as np
import torch

from gaussianavatars_b200 import synthetic as syn
from oracle import binding as ob

RAW = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
NARROW = 0.8
DOLLY = 0.1
VIEW_NAMES = ("base", "narrow", "dolly", "mirror", "repeat", "bad_fov")
KS = (1, 2, 3, 6)


def _signed_permutation(g):
    perm = torch.randperm(3, generator=g).numpy()
    sign = np.where(torch.rand(3, generator=g).numpy() < 0.5, -1.0, 1.0)
    Q = np.zeros((3, 3))
    Q[perm, np.arange(3)] = sign
    return Q


def _random_rotation(g):
    q, r = np.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64).numpy())
    return q * np.sign(np.diag(r))[None, :]


def bind(sc, seed=0, n_empty=3, hot=66):
    """Mesh-bound raw parameters reproducing the activated scene `sc` (see the module docstring).  Returns a dict:
    params (RAW + int32 binding), verts (V,3) float32, faces (F,3) int64, exact (F,) bool, and the scene's W, H,
    sh_degree, bg, name, cam and its activated tensors under "scene"."""
    g = torch.Generator().manual_seed(1000 + seed)
    x = sc["means3D"].double().numpy()
    P = x.shape[0]
    n_used = max(1, min(P // 6, 24))
    binding = torch.randint(0, n_used, (P,), generator=g).numpy()
    if P > hot + 8:
        binding[torch.randperm(P, generator=g).numpy()[:hot]] = 0
    F = n_used + n_empty
    empty = set((torch.randperm(F - 1, generator=g).numpy()[:n_empty] + 1).tolist())   # between used faces
    used = np.array([f for f in range(F) if f not in empty], np.int64)
    binding = used[binding]

    verts, exact = [], np.zeros(F, bool)
    span = float(np.abs(x).max()) if P else 1.0
    for f in range(F):
        mine = x[binding == f]
        target = mine.mean(0) if mine.size else torch.randn(3, generator=g, dtype=torch.float64).numpy() * 0.3 * span
        if f % 2 == 0:
            exact[f] = True
            Q = _signed_permutation(g)
            L = 2.0 ** int(torch.randint(-1, 2, (1,), generator=g))
            v0 = np.round((target - L * (Q[:, 0] + Q[:, 1]) / 3) * 1024) / 1024
        else:
            Q = _random_rotation(g)
            L = 0.5 + 1.5 * float(torch.rand(1, generator=g))
            off = 0.3 * (2 * torch.rand(3, generator=g, dtype=torch.float64).numpy() - 1)
            v0 = target + off - L * (Q[:, 0] + Q[:, 1]) / 3
        verts += [v0, v0 + L * Q[:, 0], v0 + L * Q[:, 1]]
    verts = torch.tensor(np.asarray(verts), dtype=torch.float32)
    faces = torch.arange(3 * F, dtype=torch.int64).reshape(F, 3)

    fr = ob.update_mesh_properties(verts.double(), faces)
    b = torch.from_numpy(binding)
    fc, fR, fs, fq = (fr[k][b] for k in ("face_center", "face_orien_mat", "face_scaling", "face_orien_quat"))
    xyz = torch.einsum("pji,pj->pi", fR, sc["means3D"].double() - fc) / fs
    fq = torch.nn.functional.normalize(fq)
    conj = torch.cat([-fq[:, 1:], fq[:, :1]], 1)                                       # xyzw
    rot = ob.quat_xyzw_to_wxyz(ob.quat_product(conj, ob.quat_wxyz_to_xyzw(sc["rotations"].double())))
    rot = rot * (0.5 + 1.5 * torch.rand(P, 1, generator=g, dtype=torch.float64))   # the chain normalises it
    o = sc["opacities"].double()
    shs = sc["shs"]
    if shs.shape[1] == 1:
        shs = torch.cat([shs, 0.3 * torch.randn(P, 3, 3, generator=g)], 1)
    f32 = lambda t: t.to(torch.float32).contiguous()  # noqa: E731
    params = dict(_xyz=f32(xyz), _rotation=f32(rot), _scaling=f32(torch.log(sc["scales"].double() / fs)),
                  _opacity=f32(torch.log(o / (1 - o))), _features_dc=f32(shs[:, :1]), _features_rest=f32(shs[:, 1:]),
                  binding=torch.from_numpy(binding.astype(np.int32)))
    scene = {k: sc[k] for k in ("means3D", "scales", "rotations", "opacities")}
    scene["shs"] = shs.contiguous()
    return dict(params=params, verts=verts, faces=faces, exact=exact, W=sc["W"], H=sc["H"], sh_degree=sc["sh_degree"],
                bg=sc["bg"], name=sc.get("name", ""), cam=sc["cam"], scene=scene, n_stack=sc.get("n_stack", 0))


def activate(bound, dtype=torch.float32, requires_grad=False):
    """The getters of oracle/binding.py on the bound parameters, in `dtype`.  Returns (act, leaves, verts): act has
    means3D, scales, rotations (wxyz), opacities, shs and cov3D (P,6) = R diag(s^2) R^T in the rasterizer's layout."""
    p = bound["params"]
    leaves = {k: p[k].to(dtype).clone().requires_grad_(requires_grad) for k in RAW}
    verts = bound["verts"].to(dtype).clone().requires_grad_(requires_grad)
    b = p["binding"].long()
    fr = ob.update_mesh_properties(verts, bound["faces"])
    act = dict(means3D=ob.get_xyz(leaves["_xyz"], b, fr["face_center"], fr["face_orien_mat"], fr["face_scaling"]),
               scales=ob.get_scaling(leaves["_scaling"], b, fr["face_scaling"]),
               rotations=ob.get_rotation(leaves["_rotation"], b, fr["face_orien_quat"]),
               opacities=ob.get_opacity(leaves["_opacity"]),
               shs=ob.get_features(leaves["_features_dc"], leaves["_features_rest"]))
    from oracle.dense64 import quat_to_R
    R = quat_to_R(act["rotations"])
    S = R @ torch.diag_embed(act["scales"] ** 2) @ R.transpose(1, 2)
    act["cov3D"] = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)
    return act, leaves, verts


def rig(bound, K):
    """The first K cameras of the six in the module docstring, as synthetic cameras; row 5's invalid field of view
    is written by `table`."""
    assert 1 <= K <= 6
    W, H = bound["W"], bound["H"]
    c0 = bound["cam"]
    fx, fy = math.degrees(c0.FoVx), math.degrees(c0.FoVy)
    nx = math.degrees(2 * math.atan(NARROW * c0.tanfovx))
    ny = math.degrees(2 * math.atan(NARROW * c0.tanfovy))
    dolly = np.eye(4, dtype=np.float32)
    dolly[2, 3] = -DOLLY
    zm = float(bound["scene"]["means3D"][:, 2].max()) + 1.0
    mirror = np.diag([-1.0, 1.0, -1.0, 1.0]).astype(np.float32)
    mirror[2, 3] = zm
    cams = [c0, syn.look_at_camera(W, H, nx, ny), syn.look_at_camera(W, H, fx, fy, w2c=dolly),
            syn.look_at_camera(W, H, fx, fy, w2c=mirror), c0, c0]
    return cams[:K]


def table(cams, device):
    """(K, 37) float32 camera table of `rig`'s cameras; row 5 (when present) with tan(FoV/2) = 0."""
    from gaussianavatars_b200.renderer import camera_table
    t = camera_table(cams, device)
    if t.shape[0] > 5:
        t[5, 35] = 0.0
    return t.contiguous()


def valid(view):
    return view != 5


def view_depth(cam, means3D):
    """float32 view-space depth of world points (the oracle's in_frustum arithmetic)."""
    V = cam.world_view_transform.numpy().reshape(16).astype(np.float32)
    m = np.asarray(means3D, np.float32)
    return V[2] * m[:, 0] + V[6] * m[:, 1] + V[10] * m[:, 2] + V[14]


def guard_out(cam, means3D):
    """Per splat: outside the 1.3 tan(FoV/2) guard band of `cam` in x or y (float32, the kernels' test)."""
    V = cam.world_view_transform.numpy().reshape(16).astype(np.float32)
    m = np.asarray(means3D, np.float32)
    tx = V[0] * m[:, 0] + V[4] * m[:, 1] + V[8] * m[:, 2] + V[12]
    ty = V[1] * m[:, 0] + V[5] * m[:, 1] + V[9] * m[:, 2] + V[13]
    tz = view_depth(cam, m)
    limx, limy = np.float32(1.3) * np.float32(cam.tanfovx), np.float32(1.3) * np.float32(cam.tanfovy)
    return (np.abs(tx / tz) > limx) | (np.abs(ty / tz) > limy)
