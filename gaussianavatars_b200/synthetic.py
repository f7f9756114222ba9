"""Synthetic workloads of BASELINE.json's shapes (no dataset / licensed FLAME assets travel to the GPU box).

Cameras restate the reference conventions (they are *inputs* of the path, not part of it):
  - `look_at_camera`   : scene/cameras.py:44-47 + utils/graphics_utils.py:38-71 (W2C^T, (P W2C)^T, centre)
  - `orbit_camera`     : utils/viewer_utils.py:20-70,127-170 as used by fps_benchmark_demo.py:21-33
    (OrbitCamera(W,H,r=1,fovy=20,'opencv'): c2w = diag(1,-1,-1), t = (0,0,r) before orbiting; projection from
    intrinsics with z_sign=+1, znear .01, zfar 10; both matrices transposed before use).
Scenes:
  - `random_splats`    : config 1 of SURVEY.md 8(d) (10k random Gaussians, identity binding)
  - `head_mesh` + `avatar_splats` : a FLAME-sized stand-in (10,144 faces; ellipsoidal "head" 0.2x0.3x0.22 m)
    with a heavy-tailed binding histogram and pre-activation parameter statistics calibrated to
    media/306/point_cloud.ply (SURVEY.md 8d: sigmoid(opacity) mean .46, ~6.6 % of splats below 1/255,
    3-sigma radius median ~13 px @1080p, ~15 tiles per splat, N ~ 1.36 M instances for 89k splats).
All generators are seeded and return CPU float32 torch tensors.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch


@dataclass
class SyntheticCamera:
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor  # (4,4) = W2C^T
    full_proj_transform: torch.Tensor   # (4,4) = (P W2C)^T
    camera_center: torch.Tensor         # (3,)
    timestep: int = 0

    @property
    def tanfovx(self):
        return math.tan(self.FoVx * 0.5)

    @property
    def tanfovy(self):
        return math.tan(self.FoVy * 0.5)

    def to(self, device):
        return SyntheticCamera(self.image_width, self.image_height, self.FoVx, self.FoVy,
                               self.world_view_transform.to(device), self.full_proj_transform.to(device),
                               self.camera_center.to(device), self.timestep)


def _projection_gs(znear, zfar, fovx, fovy):
    """utils/graphics_utils.py:51-71."""
    tx, ty = math.tan(fovx / 2), math.tan(fovy / 2)
    top, right = ty * znear, tx * znear
    P = np.zeros((4, 4), np.float32)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def look_at_camera(W, H, fovx_deg, fovy_deg, w2c: Optional[np.ndarray] = None, znear=0.01, zfar=100.0):
    w2c = np.eye(4, dtype=np.float32) if w2c is None else np.asarray(w2c, np.float32)
    fovx, fovy = math.radians(fovx_deg), math.radians(fovy_deg)
    wv = torch.tensor(w2c).transpose(0, 1).contiguous()
    proj = torch.tensor(_projection_gs(znear, zfar, fovx, fovy)).transpose(0, 1)
    full = (wv.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    center = wv.inverse()[3, :3].contiguous()
    return SyntheticCamera(W, H, fovx, fovy, wv, full, center)


def orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=0.0, elevation_deg=0.0, znear=0.01, zfar=10.0):
    focal = H / (2 * np.tan(np.radians(fovy_deg) / 2))
    fovx_deg = np.degrees(2 * np.arctan(W / (2 * focal)))
    pose = np.eye(4, dtype=np.float32)
    pose[2, 3] += r
    az, el = np.radians(azimuth_deg), np.radians(elevation_deg)
    Ry = np.array([[np.cos(az), 0, np.sin(az)], [0, 1, 0], [-np.sin(az), 0, np.cos(az)]], np.float32)
    Rx = np.array([[1, 0, 0], [0, np.cos(el), -np.sin(el)], [0, np.sin(el), np.cos(el)]], np.float32)
    rot = np.eye(4, dtype=np.float32)
    rot[:3, :3] = Ry @ Rx
    pose = rot @ pose
    pose[:, [1, 2]] *= -1  # opencv convention
    cx, cy = W // 2, H // 2
    proj = np.zeros((4, 4))
    proj[0, 0] = focal * 2 / W
    proj[1, 1] = focal * 2 / H
    proj[0, 2] = (W - 2 * cx) / W
    proj[1, 2] = (H - 2 * cy) / H
    proj[2, 2] = (zfar + znear) / (zfar - znear)
    proj[2, 3] = -2 * zfar * znear / (zfar - znear)
    proj[3, 2] = 1.0
    w2c = np.linalg.inv(pose)
    full = proj @ w2c
    return SyntheticCamera(W, H, float(np.radians(fovx_deg)), float(np.radians(fovy_deg)),
                           torch.tensor(w2c).float().T.contiguous(), torch.tensor(full).float().T.contiguous(),
                           torch.tensor(pose[:3, 3]).float().contiguous())


def random_splats(P=10_000, seed=0, sh_degree=0, max_sh_degree=None) -> Dict[str, torch.Tensor]:
    """Config 1: pre-activation parameters of P random Gaussians in front of an identity-view camera."""
    g = torch.Generator().manual_seed(seed)
    M = ((max_sh_degree if max_sh_degree is not None else sh_degree) + 1) ** 2
    xyz = torch.rand(P, 3, generator=g) * 2 - 1
    xyz[:, 2] = xyz[:, 2] * 2 + 4  # z in [2,6]
    xyz[:, :2] *= 2.0
    scaling = math.log(0.03) + 0.5 * torch.randn(P, 3, generator=g)
    rotation = torch.randn(P, 4, generator=g)
    opacity = 2.0 * torch.randn(P, 1, generator=g)
    f_dc = torch.randn(P, 1, 3, generator=g)
    f_rest = 0.3 * torch.randn(P, M - 1, 3, generator=g)
    return dict(_xyz=xyz, _scaling=scaling, _rotation=rotation, _opacity=opacity, _features_dc=f_dc,
                _features_rest=f_rest)


def head_mesh(n_lat=52, n_lon=98, seed=0):
    """Closed ellipsoidal stand-in for the FLAME head: 2*n_lon*(n_lat-1) = 9,996 + jitter faces ~ FLAME's 10,144.
    Returns verts (V,3) float32 centred at the origin and faces (F,3) int64."""
    g = np.random.default_rng(seed)
    rx, ry, rz = 0.105, 0.16, 0.11
    verts = [(0.0, ry, 0.0)]
    for i in range(1, n_lat):
        th = math.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * math.pi * j / n_lon
            verts.append((rx * math.sin(th) * math.cos(ph), ry * math.cos(th), rz * math.sin(th) * math.sin(ph)))
    verts.append((0.0, -ry, 0.0))
    verts = np.asarray(verts, np.float32)
    verts[1:-1] += g.normal(0, 2e-4, size=(len(verts) - 2, 3)).astype(np.float32)
    faces = []
    for j in range(n_lon):
        faces.append((0, 1 + (j + 1) % n_lon, 1 + j))
    for i in range(n_lat - 2):
        a, b = 1 + i * n_lon, 1 + (i + 1) * n_lon
        for j in range(n_lon):
            jn = (j + 1) % n_lon
            faces.append((a + j, a + jn, b + j))
            faces.append((a + jn, b + jn, b + j))
    last = len(verts) - 1
    a = 1 + (n_lat - 2) * n_lon
    for j in range(n_lon):
        faces.append((last, a + j, a + (j + 1) % n_lon))
    return torch.tensor(verts), torch.tensor(np.asarray(faces, np.int64))


def pose_mesh(verts: torch.Tensor, timestep: int):
    """Documented synthetic per-timestep motion (the licensed FLAME LBS is unavailable): a small rigid head turn
    plus a jaw-like shear of the lower third."""
    t = float(timestep)
    yaw, pitch = 0.15 * math.sin(0.37 * t), 0.08 * math.sin(0.23 * t + 1.0)
    Ry = torch.tensor([[math.cos(yaw), 0, math.sin(yaw)], [0, 1, 0], [-math.sin(yaw), 0, math.cos(yaw)]])
    Rx = torch.tensor([[1, 0, 0], [0, math.cos(pitch), -math.sin(pitch)], [0, math.sin(pitch), math.cos(pitch)]])
    v = verts @ (Ry @ Rx).T.to(verts)
    jaw = torch.clamp((-v[:, 1] - 0.04) / 0.1, 0, 1) * (0.01 * (1 + math.sin(0.5 * t)))
    v = v.clone()
    v[:, 1] -= jaw
    return v


FLAME_JOINT_CENTRES = np.array([[0.0, -0.12, -0.02], [0.0, -0.10, 0.0], [0.0, -0.06, 0.05], [0.035, 0.03, 0.09],
                                [-0.035, 0.03, 0.09]], np.float64)   # root, neck, jaw, eyes


def _smooth_fields(x: np.ndarray, n: int, rng, scale: float, n_waves: int = 12) -> np.ndarray:
    """n smooth displacement fields over the points x (V,3): random mixtures of low-frequency plane waves.
    Returns (V, 3, n)."""
    omega = rng.normal(0, 12.0, size=(n_waves, 3))
    phase = rng.uniform(0, 2 * np.pi, size=n_waves)
    phi = np.sin(x @ omega.T + phase)                                  # (V, n_waves)
    coef = rng.normal(0, scale / np.sqrt(n_waves / 2), size=(n_waves, 3 * n))
    return (phi @ coef).reshape(x.shape[0], 3, n)


def flame_like_assets(seed: int = 0, n_shape: int = 300, n_expr: int = 100) -> Dict[str, torch.Tensor]:
    """FLAME-shaped assets on `head_mesh()` (the licensed model is not available): smooth shape / expression fields
    scaled so that parameters of the demo's magnitudes (|shape| < 1, |expr| < 3) move the mesh by millimetres to
    centimetres, small pose correctives, a J_regressor of local averages around a root, neck, jaw and two eyes, and
    partition-of-unity skinning weights.  Buffer layouts of the reference FlameHead: v_template (V,3), shapedirs
    (V,3,n_shape+n_expr), posedirs (36,3V), J_regressor (5,V), parents [-1,0,1,1,1], lbs_weights (V,5), faces (F,3)."""
    rng = np.random.default_rng(seed)
    verts, faces = head_mesh()
    x = verts.numpy().astype(np.float64)
    V = x.shape[0]
    shapedirs = np.concatenate([_smooth_fields(x, n_shape, rng, 1e-3), _smooth_fields(x, n_expr, rng, 1.5e-3)], axis=2)
    posedirs = _smooth_fields(x, 36, rng, 2e-3).transpose(2, 0, 1).reshape(36, 3 * V)
    d2 = ((x[None, :, :] - FLAME_JOINT_CENTRES[:, None, :]) ** 2).sum(-1)   # (5, V)
    J_regressor = np.exp(-d2 / (2 * 0.03 ** 2))
    J_regressor /= J_regressor.sum(1, keepdims=True)
    logits = -d2.T / (2 * 0.05 ** 2)
    w = np.exp(logits - logits.max(1, keepdims=True))
    lbs_weights = w / w.sum(1, keepdims=True)
    f32 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32)   # noqa: E731
    return dict(v_template=verts.clone(), shapedirs=f32(shapedirs), posedirs=f32(posedirs), J_regressor=f32(J_regressor),
                parents=torch.tensor([-1, 0, 1, 1, 1], dtype=torch.long), lbs_weights=f32(lbs_weights), faces=faces,
                n_shape=n_shape, n_expr=n_expr)


def flame_like_sequence(T: int, seed: int = 0, V: Optional[int] = None, n_shape: int = 300,
                        n_expr: int = 100) -> Dict[str, torch.Tensor]:
    """A reference-style `flame_param` dict (scene/flame_gaussian_model.py:61-71) with smooth per-timestep tracks of
    the demo's magnitudes: expression (T,n_expr), rotation / neck / jaw (T,3), eyes (T,6), translation (T,3); a
    fixed shape (n_shape,) and static offset (1,V,3); dynamic offsets (T,V,3) of zeros (unused by FLAME's forward)."""
    rng = np.random.default_rng(seed)
    V = V if V is not None else head_mesh()[0].shape[0]
    ts = np.arange(T, dtype=np.float64)[:, None]

    def track(n, amp):
        f = rng.uniform(0.05, 0.4, size=(1, n))
        p = rng.uniform(0, 2 * np.pi, size=(1, n))
        return amp * np.sin(f * ts + p) * rng.uniform(0.3, 1.0, size=(1, n))

    f32 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32)   # noqa: E731
    jaw = track(3, 0.03)
    jaw[:, 0] = 0.12 * (1 + np.sin(0.3 * ts[:, 0])) / 2
    return dict(shape=f32(rng.normal(0, 0.3, size=n_shape)), expr=f32(track(n_expr, 1.2)),
                rotation=f32(track(3, 0.15)), neck_pose=f32(track(3, 0.05)), jaw_pose=f32(jaw),
                eyes_pose=f32(track(6, 0.06)), translation=f32(track(3, 0.008)),
                static_offset=f32(rng.normal(0, 5e-4, size=(1, V, 3))), dynamic_offset=torch.zeros(T, V, 3))


SIZE0, SIZE_SIG = 0.19, 0.85


def avatar_splats(P=100_000, n_faces=10_144, seed=0, sh_degree=3, scale_gain=1.0) -> Dict[str, torch.Tensor]:
    """Bound splats with media/306-like statistics.  `binding` is int32 with a heavy tail (a few faces own
    thousands of splats -- hair/teeth in the real avatar)."""
    g = torch.Generator().manual_seed(seed)
    M = (sh_degree + 1) ** 2
    # heavy-tailed face weights: log-normal + a handful of hot faces
    wts = torch.exp(1.0 * torch.randn(n_faces, generator=g))
    hot = torch.randint(0, n_faces, (12,), generator=g)
    wts[hot] *= 80.0
    binding = torch.multinomial(wts / wts.sum(), P, replacement=True, generator=g).to(torch.int32)
    # every face owns at least one splat for P >= n_faces (the reference never leaves a face empty)
    if P >= n_faces:
        binding[:n_faces] = torch.arange(n_faces, dtype=torch.int32)
    xyz = torch.randn(P, 3, generator=g) * torch.tensor([0.6, 0.6, 0.25])  # local (face) units
    # splat size: clipped log-normal body (radius quantiles of media/306: median 13 px, p90 43, p99 79, max 116 @1080p)
    size = torch.clamp(torch.randn(P, 1, generator=g), -2.5, 1.9)
    jitter = torch.clamp(torch.randn(P, 3, generator=g), -2.0, 2.0)
    scaling = math.log(SIZE0 * scale_gain) + SIZE_SIG * size + 0.35 * jitter
    scaling[:, 2] -= 0.7  # flattened along the face normal
    degenerate = torch.rand(P, generator=g) < 0.003
    scaling[degenerate] = -40.0  # exp -> ~4e-18: the radius-0 / tiny path
    rotation = torch.randn(P, 4, generator=g) * (0.5 + 2.0 * torch.rand(P, 1, generator=g))  # unnormalised raw
    opacity = -0.4 + 3.0 * torch.randn(P, 1, generator=g)
    dead = torch.rand(P, generator=g) < 0.05
    opacity[dead] = -7.0  # sigmoid < 1/255: can never contribute, must keep radii>0
    f_dc = 0.8 * torch.randn(P, 1, 3, generator=g)
    f_rest = 0.08 * torch.randn(P, M - 1, 3, generator=g)
    return dict(_xyz=xyz, _scaling=scaling, _rotation=rotation, _opacity=opacity, _features_dc=f_dc,
                _features_rest=f_rest, binding=binding)
