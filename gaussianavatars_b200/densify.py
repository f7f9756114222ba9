"""densify_and_prune on the device (SURVEY.md 8f rank 3): one gather over the six parameter arrays and their Adam
moments instead of the reference's mask-index / torch.cat sequence (scene/gaussian_model.py:334-519).

    densify_arrays(...)       tensors in, tensors out (what the tests and other frameworks call)
    add_densification_stats(model, viewspace_points, radii)
                              train.py:197 + the reference's add_densification_stats in one launch, no host wait
    densify_and_prune(model)  the reference's method on an object with the reference's attribute names
                              (_xyz ... _rotation, optimizer with named groups, xyz_gradient_accum, denom,
                              max_radii2D, percent_dense, binding, binding_counter, face_scaling): parameters are
                              replaced by new nn.Parameters inside the optimizer exactly as the reference does it,
                              so `optimizer.state_dict()` checkpoints keep working.
No CPU / eager fallback: raises when the library is missing or a tensor is not a CUDA float32 tensor.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import torch

from . import _native as N

ORDER = ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest")   # array order of the C structs
ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
        "scaling": "_scaling", "rotation": "_rotation"}


def _c(t: Optional[torch.Tensor], what: str, device, dtype=torch.float32):
    if t is None:
        return None
    if t.device != device or t.dtype != dtype:
        raise TypeError(f"{what} must be a {dtype} tensor on {device} (gaussianavatars_b200 has no CPU / eager fallback)")
    return t if t.is_contiguous() else t.contiguous()


def densify_arrays(params: Dict[str, torch.Tensor], state: Dict[str, Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]],
                   xyz_gradient_accum: torch.Tensor, denom: torch.Tensor, max_grad: float, min_opacity: float, extent: float,
                   max_screen_size: Optional[float], percent_dense: float, binding: Optional[torch.Tensor] = None,
                   binding_counter: Optional[torch.Tensor] = None, face_scaling: Optional[torch.Tensor] = None,
                   noise: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None):
    """params: name -> tensor for the names of ORDER (reference group names); state: name -> (exp_avg, exp_avg_sq) or
    (None, None).  noise: optional (2 S, 3) standard-normal tensor for the split children (S = number of split
    parents; drawn here with `generator` when absent).  Returns (params', state', binding', binding_counter', info)."""
    xyz = params["xyz"]
    device = xyz.device
    if device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    P = xyz.shape[0]
    keep = []

    def ptr(t):
        if t is None:
            return None
        keep.append(t)
        return t.data_ptr()

    a = N.DensifyArgs()
    a.abi_version, a.P = N.ABI_VERSION, P
    p = {n: _c(params[n].detach(), n, device) for n in ORDER}
    a.sh_rest_width = p["f_rest"][0].numel() if P > 0 else int(torch.tensor(p["f_rest"].shape[1:]).prod())
    a.grad_threshold, a.min_opacity, a.extent = float(max_grad), float(min_opacity), float(extent)
    a.percent_dense = float(percent_dense)
    a.max_screen_size = float(max_screen_size) if max_screen_size else -1.0
    a.xyz, a.rotation, a.scaling, a.opacity = ptr(p["xyz"]), ptr(p["rotation"]), ptr(p["scaling"]), ptr(p["opacity"])
    a.f_dc, a.f_rest = ptr(p["f_dc"]), ptr(p["f_rest"])
    st = {}
    for k, n in enumerate(ORDER):
        m, v = state.get(n, (None, None))
        m, v = _c(m, n + ".exp_avg", device), _c(v, n + ".exp_avg_sq", device)
        st[n] = (m, v)
        a.exp_avg[k], a.exp_avg_sq[k] = ptr(m), ptr(v)
    a.xyz_gradient_accum = ptr(_c(xyz_gradient_accum.reshape(-1), "xyz_gradient_accum", device))
    a.denom = ptr(_c(denom.reshape(-1), "denom", device))
    F = 0
    b32 = None
    if binding is not None:
        b32 = binding if binding.dtype == torch.int32 else binding.to(torch.int32)
        b32 = _c(b32, "binding", device, torch.int32)
        cnt = binding_counter if binding_counter.dtype == torch.int32 else binding_counter.to(torch.int32)
        cnt = _c(cnt, "binding_counter", device, torch.int32)
        fs = _c(face_scaling.reshape(-1), "face_scaling", device)
        F = cnt.shape[0]
        a.num_faces, a.binding, a.binding_counter, a.face_scaling = F, ptr(b32), ptr(cnt), ptr(fs)
    scratch = torch.empty(int(N.lib().gab200_densify_scratch_bytes(P, F)) + 256, dtype=torch.uint8, device=device)
    a.scratch = ptr(scratch)
    totals = torch.zeros(4, dtype=torch.int32).pin_memory()
    a.totals_host = totals.data_ptr()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        # extent and percent_dense in double: the thresholds are rounded to float32 once, as the reference rounds them
        N.check(N.lib().gab200_densify_plan_f64(C.byref(a), float(extent), float(percent_dense), C.c_void_p(stream)),
                "gab200_densify_plan_f64")
        n_o, n_c, n_ch, S = (int(x) for x in totals.tolist())
        P2 = n_o + n_c + 2 * n_ch
        if noise is None:
            noise = torch.randn((2 * S, 3), dtype=torch.float32, device=device, generator=generator)
        noise = _c(noise, "noise", device)
        if noise.shape[0] != 2 * S:
            raise ValueError(f"noise must have {2 * S} rows (2 per split parent), got {noise.shape[0]}")
        o = N.DensifyOut()
        o.P_out, o.n_child_rows = P2, 2 * n_ch
        out_p = {n: torch.empty((P2,) + tuple(p[n].shape[1:]), dtype=torch.float32, device=device) for n in ORDER}
        o.xyz, o.rotation, o.scaling, o.opacity = (out_p[n].data_ptr() for n in ("xyz", "rotation", "scaling", "opacity"))
        o.f_dc, o.f_rest = out_p["f_dc"].data_ptr(), out_p["f_rest"].data_ptr()
        out_s = {}
        for k, n in enumerate(ORDER):
            m, v = st[n]
            om = torch.empty_like(out_p[n]) if m is not None else None
            ov = torch.empty_like(out_p[n]) if v is not None else None
            out_s[n] = (om, ov)
            o.exp_avg[k], o.exp_avg_sq[k] = N.ptr(om), N.ptr(ov)
        b_out = c_out = None
        if binding is not None:
            b_out = torch.empty(P2, dtype=torch.int32, device=device)
            c_out = torch.empty(F, dtype=torch.int32, device=device)
            o.binding, o.binding_counter = b_out.data_ptr(), c_out.data_ptr()
        src = torch.empty(max(P2, 1), dtype=torch.int32, device=device)
        kind = torch.empty(max(P2, 1), dtype=torch.uint8, device=device)
        nrow = torch.empty(max(n_ch, 1), dtype=torch.int32, device=device)
        o.noise, o.src_scratch, o.kind_scratch, o.noise_row_scratch = noise.data_ptr(), src.data_ptr(), kind.data_ptr(), \
            nrow.data_ptr()
        N.check(N.lib().gab200_densify_apply(C.byref(a), C.byref(o), C.c_void_p(stream)), "gab200_densify_apply")
    info = dict(kept=n_o, cloned=n_c, split_children=2 * n_ch, split_parents=S, P_in=P, P_out=P2)
    return out_p, out_s, b_out, c_out, info


@torch.no_grad()
def densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size, noise=None, generator=None):
    """GaussianModel.densify_and_prune (scene/gaussian_model.py:503-519) on `model`, in place."""
    opt = model.optimizer
    groups = {g["name"]: g for g in opt.param_groups if g.get("name") in ATTR}
    params = {n: groups[n]["params"][0] for n in ATTR}
    state = {}
    for n, prm in params.items():
        s = opt.state.get(prm, None)
        state[n] = (s["exp_avg"], s["exp_avg_sq"]) if s else (None, None)
    binding = getattr(model, "binding", None)
    out_p, out_s, b_out, c_out, info = densify_arrays(
        params, state, model.xyz_gradient_accum, model.denom, max_grad, min_opacity, extent, max_screen_size,
        model.percent_dense, binding, getattr(model, "binding_counter", None) if binding is not None else None,
        getattr(model, "face_scaling", None) if binding is not None else None, noise=noise, generator=generator)
    for n, g in groups.items():
        old = g["params"][0]
        new = torch.nn.Parameter(out_p[n].requires_grad_(True))
        stored = opt.state.pop(old, None)
        if stored is not None:
            stored["exp_avg"], stored["exp_avg_sq"] = out_s[n]
            opt.state[new] = stored
        g["params"][0] = new
        setattr(model, ATTR[n], new)
    P2, dev = info["P_out"], out_p["xyz"].device
    model.xyz_gradient_accum = torch.zeros((P2, 1), device=dev)
    model.denom = torch.zeros((P2, 1), device=dev)
    model.max_radii2D = torch.zeros((P2,), device=dev)
    if binding is not None:
        model.binding = b_out.to(binding.dtype)
        model.binding_counter = c_out.to(model.binding_counter.dtype)
    return info


@torch.no_grad()
def add_densification_stats(model, viewspace_points: torch.Tensor, radii: torch.Tensor,
                            skip_flag: Optional[torch.Tensor] = None):
    """What train.py:197 and GaussianModel.add_densification_stats (scene/gaussian_model.py:517-519) do after every
    rendered frame, in place and in one launch: for every splat with radii > 0,
    `max_radii2D = max(max_radii2D, radii)`, `xyz_gradient_accum += ||viewspace_points.grad[:, :2]||`, `denom += 1`.
    The reference indexes with the boolean `visibility_filter` twice (a host wait each); this reads `radii` directly.
    `model` carries the statistics densify_and_prune consumes: xyz_gradient_accum (P, 1), denom (P, 1),
    max_radii2D (P,), float32 on the device.  `viewspace_points` is the render's `viewspace_points` after backward
    (its `.grad` is read).  skip_flag: optional int32 device tensor; non-zero when the launch executes = no change
    (graph.GraphedFrame passes its instance-overflow flag).  Capturable into a CUDA graph."""
    g = viewspace_points.grad
    if g is None:
        raise ValueError("viewspace_points has no gradient: call it after backward")
    device = g.device
    if device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    P = radii.shape[0] if radii.dim() == 1 else -1
    if P < 0 or radii.dtype != torch.int32 or radii.device != device:
        raise TypeError(f"radii must be a (P,) int32 tensor on {device}")
    if tuple(g.shape) != (P, 3) or g.dtype != torch.float32:
        raise ValueError(f"viewspace_points.grad must be a float32 ({P}, 3) tensor, got {tuple(g.shape)} {g.dtype}")
    stats = []
    for name, shape in (("xyz_gradient_accum", (P, 1)), ("denom", (P, 1)), ("max_radii2D", (P,))):
        t = getattr(model, name, None)
        if t is None or tuple(t.shape) != shape or t.dtype != torch.float32 or t.device != device \
                or not t.is_contiguous():
            got = None if t is None else (tuple(t.shape), t.dtype, str(t.device))
            raise ValueError(f"model.{name} must be a contiguous float32 {shape} tensor on {device} (P = {P} "
                             f"splats rendered), got {got}")
        stats.append(t)
    if skip_flag is not None and (skip_flag.device != device or skip_flag.dtype != torch.int32):
        raise TypeError(f"skip_flag must be an int32 tensor on {device}")
    g = g if g.is_contiguous() else g.contiguous()
    r = radii if radii.is_contiguous() else radii.contiguous()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        N.check(N.lib().gab200_densify_stats(P, g.data_ptr(), r.data_ptr(), *(t.data_ptr() for t in stats),
                                             N.ptr(skip_flag), C.c_void_p(stream)), "gab200_densify_stats")
