"""FLAME head posing on the device: blendshapes and linear blend skinning, forward and backward, for one timestep
(include/gab200_rasterizer.h gab200_flame_*).  Replaces the eager `FlameHead.forward` + `lbs`
(flame_model/flame.py:485-558, flame_model/lbs.py:25-304) that `select_mesh_by_timestep`
(scene/flame_gaussian_model.py:117-135) runs every training iteration, and its autograd.

    lbs = FlameLBS.from_flame_head(gaussians.flame_model)         # the reference's finished FlameHead (teeth added)
    verts, verts_cano = flame_pose(lbs, gaussians.flame_param, timestep)
    for group in flame_param_groups(gaussians.flame_param):       # training_setup, scene/flame_gaussian_model.py:174-207
        optimizer.add_param_group(group)

What the reference's call does and this one reproduces: `shape` and `static_offset` are constants (their optimizer
groups are commented out; they are folded into prepared constants once per change), `dynamic_offset` is accepted by
FlameHead.forward and never used (so there is no argument for it), the gradient of each per-timestep tensor is the
full (T, .) tensor with one non-zero row (so Adam steps every row, as the reference's does), and the translation is
added after skinning.  No CPU or eager fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Union

import torch

from . import _native as N

_POSED = ("expr", "rotation", "neck_pose", "jaw_pose", "eyes_pose", "translation")
_WIDTH = {"rotation": 3, "neck_pose": 3, "jaw_pose": 3, "eyes_pose": 6, "translation": 3}


def _check_kinematics(parents, n_joints: int):
    """FLAME's kinematic layout only: 5 joints, parents[0] = -1, 0 <= parents[i] < i."""
    p = [int(x) for x in parents]
    if n_joints != N.FLAME_J or len(p) != N.FLAME_J:
        raise ValueError(f"FLAME has {N.FLAME_J} joints (root, neck, jaw, two eyes); got {n_joints}")
    if p[0] != -1 or any(not 0 <= p[i] < i for i in range(1, len(p))):
        raise ValueError(f"parents must be topologically ordered with parents[0] = -1, got {p}")
    return p


class FlameLBS:
    """The FLAME model's buffers on the device plus the constants prepared from `shape` and `static_offset`.
    Build it with `from_arrays` or `from_flame_head`."""

    def __init__(self, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, faces, n_shape: int,
                 n_expr: int, device=None):
        V = int(v_template.shape[0])
        n_shape, n_expr = int(n_shape), int(n_expr)
        J = int(J_regressor.shape[0])
        self.parents = _check_kinematics(parents, J)
        want = {"v_template": (v_template, (V, 3)), "shapedirs": (shapedirs, (V, 3, n_shape + n_expr)),
                "posedirs": (posedirs, (N.FLAME_POSE_BASIS, 3 * V)), "J_regressor": (J_regressor, (J, V)),
                "lbs_weights": (lbs_weights, (V, J))}
        for name, (t, shape) in want.items():
            if tuple(t.shape) != shape:
                raise ValueError(f"{name} must have shape {shape} (n_shape={n_shape}, n_expr={n_expr}), "
                                 f"got {tuple(t.shape)}")
        if n_shape < 0 or not 0 <= n_expr <= N.FLAME_MAX_EXPR:
            raise ValueError(f"n_shape must be >= 0 and n_expr in [0, {N.FLAME_MAX_EXPR}] (FLAME's expression "
                             f"space), got {n_shape}, {n_expr}")
        device = torch.device(device if device is not None else v_template.device)
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: FlameLBS lives on a CUDA device")
        f32 = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()   # noqa: E731
        self.device = device
        self.V, self.n_shape, self.n_expr = V, n_shape, n_expr
        self.v_template, self.shapedirs, self.posedirs = f32(v_template), f32(shapedirs), f32(posedirs)
        self.J_regressor, self.lbs_weights = f32(J_regressor), f32(lbs_weights)
        self.faces = faces.to(device=device, dtype=torch.long).contiguous()
        a = N.FlameAssets()
        a.abi_version, a.V, a.n_shape, a.n_expr, a.J = N.ABI_VERSION, V, n_shape, n_expr, J
        for i, p in enumerate(self.parents):
            a.parents[i] = p
        a.v_template, a.shapedirs, a.posedirs = (self.v_template.data_ptr(), self.shapedirs.data_ptr(),
                                                 self.posedirs.data_ptr())
        a.J_regressor, a.lbs_weights = self.J_regressor.data_ptr(), self.lbs_weights.data_ptr()
        self._assets = a
        nbytes = int(N.lib().gab200_flame_scratch_bytes(V, n_expr))
        self.scratch = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self._prepared = None   # (shape tensor, its _version, static_offset tensor or None, its _version)

    @classmethod
    def from_arrays(cls, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, faces, n_shape: int,
                    n_expr: int, device=None) -> "FlameLBS":
        """Arrays in the reference FlameHead buffer layouts: v_template (V,3), shapedirs (V,3,n_shape+n_expr),
        posedirs (36,3V) (flame.py:117-119), J_regressor (5,V), parents (5,) with parents[0] = -1, lbs_weights (V,5),
        faces (F,3)."""
        return cls(v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, faces, n_shape, n_expr, device)

    @classmethod
    def from_flame_head(cls, module) -> "FlameLBS":
        """Reads the buffers of the reference's `FlameHead` (after add_teeth) and its n_shape_params / n_expr_params."""
        return cls(module.v_template, module.shapedirs, module.posedirs, module.J_regressor, module.parents.tolist(),
                   module.lbs_weights, module.faces, module.n_shape_params, module.n_expr_params,
                   module.v_template.device)

    def prepare(self, shape: torch.Tensor, static_offset: Optional[torch.Tensor] = None):
        """Folds `shape` (n_shape,) and `static_offset` ((1,V,3) as the reference stores it, or (V,3); None = 0)
        into the prepared constants.  Runs only when either tensor is a different object or was changed in place."""
        for name, t in (("shape", shape), ("static_offset", static_offset)):
            if t is not None and t.requires_grad:
                raise ValueError(f"flame_param['{name}'] requires grad, but it is a constant here as in the reference "
                                 "(its optimizer group is commented out)")
        p = self._prepared
        if p is not None and p[0] is shape and p[1] == shape._version and p[2] is static_offset and \
                p[3] == (None if static_offset is None else static_offset._version):
            return
        if shape.numel() != self.n_shape:
            raise ValueError(f"shape must have {self.n_shape} entries, got {tuple(shape.shape)}")
        s = shape.detach().to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        so = None
        if static_offset is not None:
            if static_offset.numel() != 3 * self.V:
                raise ValueError(f"static_offset must be (1,{self.V},3) or ({self.V},3), got {tuple(static_offset.shape)}")
            so = static_offset.detach().to(device=self.device, dtype=torch.float32).reshape(self.V, 3).contiguous()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            N.check(N.lib().gab200_flame_prepare(C.byref(self._assets), s.data_ptr(), N.ptr(so),
                                                 self.scratch.data_ptr(), C.c_void_p(stream)), "gab200_flame_prepare")
        self._prepared = (shape, shape._version, static_offset,
                          None if static_offset is None else static_offset._version)

    def state_key(self):
        """What a captured graph bakes in of this model: the prepared constants' source tensors and versions."""
        p = self._prepared
        return None if p is None else (id(p[0]), p[1], id(p[2]), p[3], self.scratch.data_ptr())


class _FlamePose(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lbs, t_dev, expr, rotation, neck_pose, jaw_pose, eyes_pose, translation):
        dev = lbs.device
        T = int(expr.shape[0])
        frame = torch.empty(N.FLAME_FRAME_FLOATS, dtype=torch.float32, device=dev)
        verts = torch.empty((1, lbs.V, 3), dtype=torch.float32, device=dev)
        cano = torch.empty((1, lbs.V, 3), dtype=torch.float32, device=dev)
        params = (expr, rotation, neck_pose, jaw_pose, eyes_pose, translation)
        a = N.FlameFrameArgs()
        a.abi_version, a.T, a.assets, a.scratch = N.ABI_VERSION, T, C.pointer(lbs._assets), lbs.scratch.data_ptr()
        a.timestep = t_dev.data_ptr()
        a.expr, a.rotation, a.neck_pose, a.jaw_pose, a.eyes_pose, a.translation = (p.data_ptr() for p in params)
        a.frame = frame.data_ptr()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            N.check(N.lib().gab200_flame_forward(C.byref(a), verts.data_ptr(), cano.data_ptr(), C.c_void_p(stream)),
                    "gab200_flame_forward")
        ctx.args, ctx.keep, ctx.lbs = a, (t_dev, frame) + params, lbs
        return verts, cano

    @staticmethod
    def backward(ctx, g_verts, g_cano):
        a, dev = ctx.args, ctx.lbs.device
        params = ctx.keep[2:]
        grads = [torch.empty_like(p) for p in params]
        gv = torch.zeros((1, ctx.lbs.V, 3), dtype=torch.float32, device=dev) if g_verts is None else g_verts.contiguous()
        gc = None if g_cano is None else g_cano.contiguous()
        out = N.FlameGrads(*(g.data_ptr() for g in grads))
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            N.check(N.lib().gab200_flame_backward(C.byref(a), gv.data_ptr(), N.ptr(gc), C.byref(out),
                                                  C.c_void_p(stream)), "gab200_flame_backward")
        return (None, None, *grads)


def _posed_params(lbs: FlameLBS, flame_param: Dict[str, torch.Tensor]):
    T = int(flame_param["expr"].shape[0])
    out = []
    for k in _POSED:
        t = flame_param[k]
        shape = (T, lbs.n_expr) if k == "expr" else (T, _WIDTH[k])
        if tuple(t.shape) != shape:
            raise ValueError(f"flame_param['{k}'] must have shape {shape}, got {tuple(t.shape)}")
        if t.device != lbs.device or t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError(f"flame_param['{k}'] must be a contiguous float32 tensor on {lbs.device}")
        out.append(t)
    return T, out


def timestep_tensor(timestep: Union[int, torch.Tensor], T: int, device) -> torch.Tensor:
    """A host int is checked against [0, T) and placed in a new device int32; a device int32 scalar is used as is
    (it is read by the kernels: out of range there leaves the outputs unspecified, memory-safe)."""
    if isinstance(timestep, torch.Tensor):
        if timestep.device != device or timestep.dtype != torch.int32 or timestep.numel() != 1:
            raise TypeError(f"a tensor timestep must be one int32 on {device}")
        return timestep
    return torch.full((1,), check_timestep(timestep, T), dtype=torch.int32, device=device)


def check_timestep(timestep, T: int) -> int:
    """A host timestep as an int, checked against [0, T)."""
    t = int(timestep)
    if not 0 <= t < T:
        raise IndexError(f"timestep {t} outside [0, {T})")
    return t


def flame_pose(lbs: FlameLBS, flame_param: Dict[str, torch.Tensor], timestep: Union[int, torch.Tensor]):
    """`FlameHead.forward(shape[None], expr[[t]], rotation[[t]], neck_pose[[t]], jaw_pose[[t]], eyes_pose[[t]],
    translation[[t]], zero_centered_at_root_node=False, return_landmarks=False, return_verts_cano=True,
    static_offset=static_offset)` for the reference's `flame_param` dict (scene/flame_gaussian_model.py:61-71,
    121-134): returns (verts (1,V,3), verts_cano (1,V,3)), differentiable w.r.t. the six per-timestep tensors.
    `timestep` is a Python int or an int32 device scalar (what a captured graph reads)."""
    lbs.prepare(flame_param["shape"], flame_param.get("static_offset"))
    T, params = _posed_params(lbs, flame_param)
    return _FlamePose.apply(lbs, timestep_tensor(timestep, T, lbs.device), *params)


def flame_param_groups(flame_param: Dict[str, torch.Tensor], pose_lr: float = 1e-5, trans_lr: float = 1e-6,
                       expr_lr: float = 1e-3):
    """The FLAME parameter groups of FlameGaussianModel.training_setup (scene/flame_gaussian_model.py:174-207;
    learning rates arguments/__init__.py:95-97), ready for `optimizer.add_param_group`.  Marks the tensors as
    requiring grad, as training_setup does."""
    pose = [flame_param[k] for k in ("rotation", "neck_pose", "jaw_pose", "eyes_pose")]
    for t in pose + [flame_param["translation"], flame_param["expr"]]:
        t.requires_grad_(True)
    return [{"params": pose, "lr": pose_lr, "name": "pose"},
            {"params": [flame_param["translation"]], "lr": trans_lr, "name": "trans"},
            {"params": [flame_param["expr"]], "lr": expr_lr, "name": "expr"}]
