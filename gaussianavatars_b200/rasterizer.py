"""Host-side mirror of the reference operator surface, backed by the sm_90a C-ABI library.

Drop-in names (the only two GaussianAvatars imports, gaussian_renderer/__init__.py:15):
    GaussianRasterizationSettings, GaussianRasterizer
with the semantics of diff_gaussian_rasterization/__init__.py of the pinned submodule (SURVEY.md 8b, Appendix B.6):
same argument names, same "exactly one of" exceptions, same outputs (color (3,H,W), radii (P,) int32), same
gradient tuple (means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, None).

New, opt-in fused surface (SURVEY.md 8b "Fused surface"): `rasterize_bound(...)` takes the RAW GaussianModel
parameters plus the per-face frame and runs scene/gaussian_model.py:113-160 inside the preprocess kernel; its
backward returns gradients for the raw parameters and for face_center / face_orien_mat / face_scaling.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _native as N


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


# Binning policy of the library (include/gab200_rasterizer.h `exact_binning`).  False (default) drops (splat, tile)
# pairs that provably contribute nothing; image, radii and gradients are unchanged.  True reproduces the
# reference's full 3-sigma bounding-square instance list (used by the key/sort parity tests).
_EXACT_BINNING = False


def set_exact_binning(flag: bool):
    global _EXACT_BINNING
    _EXACT_BINNING = bool(flag)


def _f32c(t: Optional[torch.Tensor], name: str, device):
    if t is None or t.numel() == 0:
        return None
    if t.device != device:
        raise ValueError(f"{name} must live on {device}, got {t.device}")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _cam(t: torch.Tensor, name: str, device):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a tensor")
    if t.device != device or t.dtype != torch.float32:
        t = t.to(device=device, dtype=torch.float32)
    return t if t.is_contiguous() else t.contiguous()


class FrameHints:
    """What one caller (one splat model) has learnt about its frames: per (device, W, H, P), the instance count of the
    last frame (the capacity the next one runs with: gab200_forward_args.binning_hint) and the depth-key range
    (depth_hint_*).  Hints never change a result, only how much of the forward is enqueued before the host learns N.
    `render()` keeps one on the model object (`pc._gab200_hints`); callers of the bare operator surface that cannot
    pass one (the reference's own render() builds a new GaussianRasterizer per frame) share `_default_hints`."""

    MAX_SHAPES = 64  # P changes at every densification: do not let the per-shape hints pile up

    def __init__(self):
        self.shapes = {}
        self.seq = 0
        self.last = None  # info dict of the last forward that used these hints

    def get(self, key):
        return self.shapes.get(key, (0, (0, 0)))

    def set_depth(self, key, depth_range):
        self.shapes[key] = (self.get(key)[0], tuple(depth_range))

    def set_capacity(self, key, capacity: int):
        self.shapes[key] = (int(capacity), self.get(key)[1])

    def put(self, key, n: int, depth_range):
        if len(self.shapes) >= self.MAX_SHAPES and key not in self.shapes:
            self.shapes.clear()
        self.shapes[key] = (min(int(n * 1.25) + 4096, 2**31 - 1), depth_range)


_default_hints = FrameHints()
_SYNC_POLICY = "late"   # "late": sync-free enqueue + end-of-call check whenever a capacity hint exists; "exact": always mid-frame


def set_sync_policy(policy: str):
    """"late" (default) or "exact" -- see include/gab200_rasterizer.h gab200_sync_mode.  Results are identical."""
    global _SYNC_POLICY
    if policy not in ("late", "exact"):
        raise ValueError("policy must be 'late' or 'exact'")
    _SYNC_POLICY = policy


def hints_of(obj) -> "FrameHints":
    """The FrameHints attached to a model object (created on first use); `_default_hints` if it cannot carry one."""
    h = getattr(obj, "_gab200_hints", None)
    if h is None:
        h = FrameHints()
        try:
            obj._gab200_hints = h
        except Exception:
            return _default_hints
    return h


def _fill_common(a: N.ForwardArgs, rs: GaussianRasterizationSettings, device, P: int, need_backward: bool,
                 cameras: Optional[torch.Tensor] = None):
    """The scalar fields and camera pointers of `a`; returns the tensors they point at.  With a (K, 37) camera table
    the views' matrices, centres and fields of view are in the table: `a`'s stay unset."""
    a.abi_version = N.ABI_VERSION
    a.P = P
    a.sh_degree = int(rs.sh_degree)
    a.image_width = int(rs.image_width)
    a.image_height = int(rs.image_height)
    a.scale_modifier = float(rs.scale_modifier)
    a.prefiltered = int(bool(rs.prefiltered))
    a.debug = int(bool(rs.debug))
    a.need_backward = int(need_backward)
    a.exact_binning = int(_EXACT_BINNING)
    if cameras is not None:
        bg = _cam(rs.bg, "bg", device)
        a.bg = bg.data_ptr()
        return (bg,)
    a.tanfovx = float(rs.tanfovx)
    a.tanfovy = float(rs.tanfovy)
    cams = (_cam(rs.bg, "bg", device), _cam(rs.viewmatrix, "viewmatrix", device),
            _cam(rs.projmatrix, "projmatrix", device), _cam(rs.campos, "campos", device))
    a.bg, a.viewmatrix, a.projmatrix, a.campos = (t.data_ptr() for t in cams)
    return cams


_KEEP_LAST = False
_last = None
_last_info = {}


def _widen_depth_range(kmin: int, kmax: int):
    """The last frame's visible depth-key range plus 1/8 of its width either side (keys are fp32 bit patterns of
    positive depths: monotonic, so a range in key space is a range in depth).  A frame that falls outside is still
    sorted correctly -- outliers share the two end buckets -- so the margin only has to keep that rare."""
    pad = max((kmax - kmin) // 8, 1 << 12)
    return max(kmin - pad, 1), min(kmax + pad, 0xFFFFFFFE)


def keep_last_state(flag: bool):
    """Parity/debug hook: retain the last forward's scratch so `export_last_binning()` can read the sorted stream."""
    global _KEEP_LAST, _last
    _KEEP_LAST = bool(flag)
    if not flag:
        _last = None


def export_last_binning():
    """(keys u64 as int64 tensor, values int32 tensor, ranges (tiles,2) int32 tensor, num_rendered) of the last forward."""
    if _last is None:
        raise RuntimeError("keep_last_state(True) was not set before the forward")
    a, st, holder, device = _last
    n = int(st.num_rendered)
    gx, gy = (a.image_width + 15) // 16, (a.image_height + 15) // 16
    keys = torch.empty((max(n, 1),), dtype=torch.int64, device=device)
    vals = torch.empty((max(n, 1),), dtype=torch.int32, device=device)
    ranges = torch.empty((gx * gy, 2), dtype=torch.int32, device=device)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        N.check(N.lib().gab200_export_binning(C.byref(a), C.byref(st), keys.data_ptr(), vals.data_ptr(),
                                              ranges.data_ptr(), C.c_void_p(stream)), "gab200_export_binning")
    return keys[:n], vals[:n], ranges, n


def last_frame_info() -> dict:
    """How the last forward on this process went: instances, capacity, depth-sort path, sync mode, attempts."""
    return dict(_last_info)


class CaptureSlot:
    """What a forward needs while its stream is being captured into a CUDA graph (GAB200_SYNC_NONE): a fixed
    capacity, a pinned host copy of the frame counters, and a sticky device flag the library raises when a replay
    overflows the capacity (graph.py owns one per captured step)."""

    def __init__(self, device, capacity: int, depth_range=(0, 0)):
        self.capacity = int(capacity)
        self.depth_range = depth_range
        self.counters = torch.zeros(N.NUM_COUNTERS, dtype=torch.int32).pin_memory()
        self.flag = torch.zeros(1, dtype=torch.int32, device=device)   # sticky: set by the library on overflow
        self.flag_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.seq = 1
        self.info = {}
        self.scratch = None   # a captured forward-only frame's own scratch (see _run_frame)


_capture_slot = None
_tls = threading.local()


def visible_of(radii: torch.Tensor):
    """The `radii > 0` mask the forward that produced `radii` wrote beside it (None if that was not the last forward
    of this thread)."""
    v = getattr(_tls, "visible", None)
    return v[1] if v is not None and v[0] == radii.data_ptr() else None


def check_tanfov(tanfov: Optional[torch.Tensor], device):
    """A camera's device field of view: a (2,) float32 tensor {tan(FoVx/2), tan(FoVy/2)} on `device`, or None."""
    if tanfov is None:
        return None
    if not isinstance(tanfov, torch.Tensor) or tanfov.device != device or tanfov.dtype != torch.float32 or \
            tanfov.numel() != 2 or not tanfov.is_contiguous():
        raise ValueError(f"tanfov must be a contiguous (2,) float32 tensor on {device}")
    return tanfov


def check_rgb8(rgb8: Optional[torch.Tensor], rs: GaussianRasterizationSettings, device, lead: tuple = ()):
    """A display-image destination: a contiguous lead + (H,W,3) uint8 tensor on `device`, or None."""
    if rgb8 is None:
        return None
    shape = lead + (int(rs.image_height), int(rs.image_width), 3)
    if not isinstance(rgb8, torch.Tensor) or rgb8.device != device or rgb8.dtype != torch.uint8 or \
            tuple(rgb8.shape) != shape or not rgb8.is_contiguous():
        raise ValueError(f"rgb8 must be a contiguous {shape} uint8 tensor on {device}")
    return rgb8


def _run_frame(a: N.ForwardArgs, device, need_backward: bool, key, hints: FrameHints, name: str, enqueue, **extra):
    """One forward through the library.  Inside a CUDA-graph capture (`_capture_slot`): the slot's fixed capacity and
    counters, no host wait.  Otherwise the capacity and depth-range hints `hints` learnt from earlier frames of shape
    `key`, updated with this frame's outcome.  enqueue(st, stream) calls the entry point; `extra` joins the info dict.
    Returns (frame state, scratch holder, info)."""
    slot = _capture_slot
    # A forward-only frame captured into a graph must own its scratch: the pooled inference buffers are shared with
    # every eager no_grad render and replaced when a larger frame comes along, so the graph's baked-in pointers would
    # be overwritten or freed.  Allocated during the capture, the scratch lives in the graph's private pool.
    cb, holder = N.begin_forward(device, need_backward or slot is not None)
    if slot is not None and not need_backward:
        slot.scratch = holder
    a.alloc_geom = a.alloc_binning = a.alloc_image = cb
    st = N.FrameState()
    if slot is not None:      # graph capture: fixed capacity, no host wait; graph.py reads slot.counters after replays
        a.sync_mode = N.SYNC_NONE
        a.binning_hint = slot.capacity
        a.depth_hint_lo, a.depth_hint_hi = slot.depth_range
        a.frame_seq = slot.seq
        a.counters_host = slot.counters.data_ptr()
        a.overflow_flag = slot.flag.data_ptr()
    else:
        a.binning_hint, (a.depth_hint_lo, a.depth_hint_hi) = hints.get(key)
        a.sync_mode = N.SYNC_LATE if (_SYNC_POLICY == "late" and a.binning_hint > 0) else N.SYNC_EXACT
        hints.seq = (hints.seq + 1) & 0x7FFFFFFF
        a.frame_seq = hints.seq
    with torch.cuda.device(device):
        n = enqueue(st, C.c_void_p(torch.cuda.current_stream(device).cuda_stream))
    N.check(n, name)
    info = dict(num_rendered=int(st.num_rendered), capacity=int(st.binning_capacity), sync_mode=int(a.sync_mode),
                depth_sort_path=int(st.depth_sort_path), attempts=int(st.attempts), **extra)
    if slot is not None:
        slot.info = info
    else:
        hints.put(key, n, _widen_depth_range(st.depth_key_min, st.depth_key_max)
                  if st.depth_key_min <= st.depth_key_max else (0, 0))
        hints.last = info
    return st, holder, info


def _run_forward(a: N.ForwardArgs, device, need_backward: bool, hints: Optional[FrameHints] = None,
                 tanfov: Optional[torch.Tensor] = None, rgb8: Optional[torch.Tensor] = None, float_image: bool = True,
                 planes: Optional[tuple] = None, cameras: Optional[torch.Tensor] = None):
    """tanfov: None (a.tanfovx / tanfovy) or the (2,) device tensor the kernels read instead
    (gab200_forward_device_fov); the backward must then be given the same tensor.
    rgb8: None, or a (H,W,3) uint8 tensor the blend writes the display image into (gab200_forward_display);
    float_image=False (with rgb8, no backward) skips the float image: the returned color is None.
    planes: None, or (alpha, depth) (1,H,W) float32 tensors the blend also fills (gab200_forward_depth_alpha).
    cameras: None (one camera, from `a`), or a checked (K, 37) table of K views (gab200_forward_views[_train]
    [_depth_alpha]; tanfov is not read): color, radii, rgb8 and planes then have a leading K, and the hints are those
    of key (device, W, H, P, K).  Only single-view frames are recorded for last_frame_info / export_last_binning."""
    global _last, _last_info
    H, W, P = a.image_height, a.image_width, a.P
    lead = () if cameras is None else (int(cameras.shape[0]),)
    color = torch.empty(lead + (3, H, W), dtype=torch.float32, device=device) if float_image else None
    radii = torch.empty(lead + (P,), dtype=torch.int32, device=device)
    visible = torch.empty(lead + (P,), dtype=torch.bool, device=device)   # radii > 0, written by the preprocess kernel
    a.out_color, a.radii, a.visibility = N.ptr(color), radii.data_ptr(), visible.data_ptr()
    _tls.visible = (radii.data_ptr(), visible)   # renderer.py hands it out as `visibility_filter`
    hints = hints if hints is not None else _default_hints
    alpha, depth = (None, None) if planes is None else (planes[0].data_ptr(), planes[1].data_ptr())

    def enqueue(st, stream):
        if cameras is not None:
            K, table = lead[0], cameras.data_ptr()
            if need_backward and planes is not None:
                return N.lib().gab200_forward_views_train_depth_alpha(C.byref(a), K, table, alpha, depth, C.byref(st),
                                                                      stream)
            if need_backward:
                return N.lib().gab200_forward_views_train(C.byref(a), K, table, C.byref(st), stream)
            if planes is not None:
                return N.lib().gab200_forward_views_depth_alpha(C.byref(a), K, table, alpha, depth, N.ptr(rgb8),
                                                                C.byref(st), stream)
            return N.lib().gab200_forward_views(C.byref(a), K, table, N.ptr(rgb8), C.byref(st), stream)
        if planes is not None:
            return N.lib().gab200_forward_depth_alpha(C.byref(a), N.ptr(tanfov), alpha, depth, N.ptr(rgb8),
                                                      C.byref(st), stream)
        if rgb8 is not None:
            return N.lib().gab200_forward_display(C.byref(a), N.ptr(tanfov), rgb8.data_ptr(), C.byref(st), stream)
        if tanfov is not None:
            return N.lib().gab200_forward_device_fov(C.byref(a), tanfov.data_ptr(), C.byref(st), stream)
        return N.lib().gab200_forward(C.byref(a), C.byref(st), stream)

    if cameras is None:
        st, holder, info = _run_frame(a, device, need_backward, (device, W, H, P), hints, "gab200_forward", enqueue)
        _last_info = info
        if _KEEP_LAST:
            # pooled (inference) scratch stays valid until the next no_grad forward on this device
            _last = (a, st, holder, device)
    else:
        st, holder, _ = _run_frame(a, device, need_backward, (device, W, H, P) + lead, hints,
                                   "gab200_forward_views_train" if need_backward else "gab200_forward_views", enqueue,
                                   views=lead[0])
    return color, radii, st, holder


def _run_backward(b: N.BackwardArgs, device, tanfov: Optional[torch.Tensor] = None,
                  plane_grads: Optional[tuple] = None, cameras: Optional[torch.Tensor] = None):
    """gab200_backward, or gab200_backward_device_fov with the tensor the forward read; plane_grads: (dL/dalpha,
    dL/ddepth), each a contiguous (1,H,W) tensor or None, of a depth_alpha frame (gab200_backward_depth_alpha).
    cameras: the (K, 37) table of a K-view frame (gab200_backward_views[_depth_alpha]; plane gradients (K,1,H,W))."""
    with torch.cuda.device(device):
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        ga, gd = (None, None) if plane_grads is None else (N.ptr(plane_grads[0]), N.ptr(plane_grads[1]))
        if cameras is not None:
            K, table = int(cameras.shape[0]), cameras.data_ptr()
            if plane_grads is not None:
                N.check(N.lib().gab200_backward_views_depth_alpha(C.byref(b), K, table, ga, gd, stream),
                        "gab200_backward_views_depth_alpha")
            else:
                N.check(N.lib().gab200_backward_views(C.byref(b), K, table, stream), "gab200_backward_views")
        elif plane_grads is not None:
            N.check(N.lib().gab200_backward_depth_alpha(C.byref(b), N.ptr(tanfov), ga, gd, stream),
                    "gab200_backward_depth_alpha")
        elif tanfov is None:
            N.check(N.lib().gab200_backward(C.byref(b), stream), "gab200_backward")
        else:
            N.check(N.lib().gab200_backward_device_fov(C.byref(b), tanfov.data_ptr(), stream), "gab200_backward")


class _RasterizeGaussians(torch.autograd.Function):
    """Reference surface (ACTIVATED inputs)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, hints=None):
        rs = raster_settings
        device = means3D.device
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
        if means3D.ndim != 2 or means3D.shape[1] != 3:
            raise RuntimeError("means3D must have dimensions (num_points, 3)")
        P = means3D.shape[0]
        need_bw = any(ctx.needs_input_grad)
        a = N.ForwardArgs()
        cams = _fill_common(a, rs, device, P, need_bw)
        a.input_mode = N.INPUT_ACTIVATED
        means3D = _f32c(means3D, "means3D", device)
        sh = _f32c(sh, "shs", device)
        colors_precomp = _f32c(colors_precomp, "colors_precomp", device)
        opacities = _f32c(opacities, "opacities", device)
        scales = _f32c(scales, "scales", device)
        rotations = _f32c(rotations, "rotations", device)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, "cov3D_precomp", device)
        a.sh_coeffs = 0 if sh is None else sh.shape[1]
        a.means3D, a.opacities = N.ptr(means3D), N.ptr(opacities)
        a.scales, a.rotations, a.cov3D_precomp = N.ptr(scales), N.ptr(rotations), N.ptr(cov3Ds_precomp)
        a.shs, a.colors_precomp = N.ptr(sh), N.ptr(colors_precomp)
        color, radii, st, holder = _run_forward(a, device, need_bw, hints)
        if need_bw:
            ctx.args, ctx.state, ctx.holder = a, st, holder
            ctx.keep = (cams, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, radii)
            ctx.M = a.sh_coeffs
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii):
        a, st = ctx.args, ctx.state
        cams, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, radii = ctx.keep
        device = means3D.device
        P, M = a.P, ctx.M
        g = grad_out_color if grad_out_color.is_contiguous() else grad_out_color.contiguous()
        e = lambda *s: torch.empty(s, dtype=torch.float32, device=device)  # noqa: E731
        d_means3D, d_means2D, d_opac = e(P, 3), e(P, 3), e(P, 1)
        d_colors = e(P, 3)
        d_sh = e(P, M, 3) if sh is not None else None
        d_scales = e(P, 3) if scales is not None else None
        d_rots = e(P, 4) if rotations is not None else None
        d_cov = e(P, 6)
        b = N.BackwardArgs()
        b.abi_version = N.ABI_VERSION
        b.fwd, b.state = C.pointer(a), C.pointer(st)
        b.dL_dout_color = g.data_ptr()
        b.dL_dmeans3D, b.dL_dmeans2D, b.dL_dopacity = d_means3D.data_ptr(), d_means2D.data_ptr(), d_opac.data_ptr()
        b.dL_dcolors, b.dL_dshs = d_colors.data_ptr(), N.ptr(d_sh)
        b.dL_dscales, b.dL_drotations, b.dL_dcov3D = N.ptr(d_scales), N.ptr(d_rots), d_cov.data_ptr()
        _run_backward(b, device)
        ctx.holder = None
        return (d_means3D, d_means2D, d_sh, d_colors if colors_precomp is not None else None, d_opac, d_scales, d_rots,
                d_cov if cov3Ds_precomp is not None else None, None, None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, hints: Optional[FrameHints] = None):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, hints)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings, hints: Optional[FrameHints] = None):
        """`hints` is an extension over the reference's constructor (optional; see FrameHints)."""
        super().__init__()
        self.raster_settings = raster_settings
        self.hints = hints

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            device = positions.device
            pos = _f32c(positions, "positions", device)
            out = torch.empty((pos.shape[0],), dtype=torch.uint8, device=device)
            view, proj = _cam(rs.viewmatrix, "viewmatrix", device), _cam(rs.projmatrix, "projmatrix", device)
            with torch.cuda.device(device):
                stream = torch.cuda.current_stream(device).cuda_stream
                N.check(N.lib().gab200_mark_visible(pos.shape[0], pos.data_ptr(), view.data_ptr(), proj.data_ptr(),
                                                    out.data_ptr(), C.c_void_p(stream)), "gab200_mark_visible")
        return out.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, depth_alpha=False):
        """The reference's (color, radii).  depth_alpha=True is refused: the alpha / depth planes are on the fused
        route, rasterize_bound(..., depth_alpha=True) or render(..., depth_alpha=True)."""
        if depth_alpha:
            raise ValueError("GaussianRasterizer (the drop-in for diff_gaussian_rasterization) returns the reference's "
                             "(color, radii) only: for the alpha and depth planes use the fused route, "
                             "rasterize_bound(..., depth_alpha=True) or render(..., depth_alpha=True)")
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, self.raster_settings, self.hints)


# ================================================================================================================
# Fused surface
# ================================================================================================================
_face_csr_cache = {}   # id(binding tensor the caller passed) -> (that tensor, its _version, F, int32 copy, CSR tuple)


def _face_csr(binding: torch.Tensor, num_faces: int, chunk: int = 16):
    """(int32 contiguous binding, face-sorted view of it for the backward's per-face reduction
    (gab200_backward_args.face_*)).  The binding only changes at densification
    (scene/gaussian_model.py:472-474,495-497), so this runs once per change.  Keyed on the caller's OWN tensor (a
    reference is kept, so its id cannot be recycled) and its in-place version: a temporary `.to(int32)` copy whose
    address the allocator reuses can never alias another model's entry."""
    key = id(binding)
    hit = _face_csr_cache.get(key)
    if hit is not None and hit[0] is binding and hit[1] == binding._version and hit[2] == num_faces:
        return hit[3], hit[4]
    b32 = binding if binding.dtype == torch.int32 and binding.is_contiguous() else binding.to(torch.int32).contiguous()
    b = b32.long()
    perm = torch.argsort(b, stable=True).to(torch.int32)
    counts = torch.bincount(b, minlength=num_faces)
    starts = torch.cumsum(counts, 0) - counts
    nchunks = (counts + chunk - 1) // chunk
    face = torch.repeat_interleave(torch.arange(num_faces, device=b.device), nchunks)
    first = torch.cumsum(nchunks, 0) - nchunks
    within = torch.arange(face.shape[0], device=b.device) - first[face]
    c_start = starts[face] + within * chunk
    c_end = torch.minimum(c_start + chunk, starts[face] + counts[face])
    out = (perm.contiguous(), face.to(torch.int32).contiguous(), c_start.to(torch.int32).contiguous(),
           c_end.to(torch.int32).contiguous())
    if len(_face_csr_cache) >= 8:
        _face_csr_cache.clear()
    _face_csr_cache[key] = (binding, binding._version, num_faces, b32, out)
    return b32, out


def _fill_bound(a: N.ForwardArgs, device, _xyz, _rotation, _scaling, _opacity, f_dc, f_rest, colors_precomp, binding,
                face_center, face_orien_mat, face_scaling):
    """The BOUND_RAW inputs of `a` from the raw model tensors and the per-face frame.  Returns the tensors `a` points
    at (keep them alive while the library may read them): (_xyz, _rotation, _scaling, _opacity, f_dc, f_rest,
    colors_precomp, binding, face_center, face_orien_mat, face_scaling), binding int32 and the rest contiguous
    float32, None where not given."""
    a.input_mode = N.INPUT_BOUND_RAW
    _xyz, _rotation = _f32c(_xyz, "_xyz", device), _f32c(_rotation, "_rotation", device)
    _scaling, _opacity = _f32c(_scaling, "_scaling", device), _f32c(_opacity, "_opacity", device)
    f_dc, f_rest = _f32c(f_dc, "_features_dc", device), _f32c(f_rest, "_features_rest", device)
    colors_precomp = _f32c(colors_precomp, "colors_precomp", device)
    a.sh_coeffs = 1 + (0 if f_rest is None else f_rest.shape[1])
    a.means3D, a.rotations, a.scales, a.opacities = _xyz.data_ptr(), _rotation.data_ptr(), _scaling.data_ptr(), \
        _opacity.data_ptr()
    a.sh_dc, a.sh_rest, a.colors_precomp = N.ptr(f_dc), N.ptr(f_rest), N.ptr(colors_precomp)
    if binding is not None:
        if binding.dtype != torch.int32 or not binding.is_contiguous():
            binding = _face_csr(binding, face_center.shape[0])[0]  # converted once per binding, not per frame
        face_center = _f32c(face_center, "face_center", device)
        face_orien_mat = _f32c(face_orien_mat, "face_orien_mat", device)
        face_scaling = _f32c(face_scaling, "face_scaling", device)
        a.binding, a.num_faces = binding.data_ptr(), face_center.shape[0]
        a.face_center, a.face_orien_mat, a.face_scaling = face_center.data_ptr(), face_orien_mat.data_ptr(), \
            face_scaling.data_ptr()
    return (_xyz, _rotation, _scaling, _opacity, f_dc, f_rest, colors_precomp, binding, face_center, face_orien_mat,
            face_scaling)


def _grad_buffer(grad_sink, P: int, M: int, device, symm_ok: bool = True):
    """One flat buffer for all per-splat parameter gradients (dist.py all-reduces it in ONE collective):
    [_xyz 3 | _rotation 4 | _scaling 3 | _opacity 1 | f_dc 3 | f_rest 3(M-1)]  = 59 floats/splat at SH3.
    It is grad_sink's symmetric gradient buffer when that is enabled, of this size and `symm_ok`, else a new tensor.
    Returns (flat, the symmetric buffer used or None, (d_xyz, d_rot, d_scale, d_opac, d_dc, d_rest or None))."""
    widths = (3, 4, 3, 1, 3, 3 * (M - 1))
    symm = getattr(grad_sink, "symm_grad", None) if grad_sink is not None else None
    if not (symm_ok and symm is not None and symm.enabled and symm.numel == P * sum(widths)):
        symm = None
    flat = symm.flat if symm is not None else torch.empty((P * sum(widths),), dtype=torch.float32, device=device)
    views, off = [], 0
    for w in widths:
        views.append(flat[off:off + P * w])
        off += P * w
    grads = (views[0].view(P, 3), views[1].view(P, 4), views[2].view(P, 3), views[3].view(P, 1),
             views[4].view(P, 1, 3), views[5].view(P, M - 1, 3) if M > 1 else None)
    return flat, symm, grads


class _RasterizeBound(torch.autograd.Function):
    """The fused route's frame: one camera from raster_settings (and `tanfov`), or with `cameras`, a checked (K, 37)
    table, the K views of one splat set, every image, radii and means2D with a leading K.  colors_precomp and the
    multicast gradient buffer are single-view only (the K-view entry points refuse both)."""

    @staticmethod
    def forward(ctx, _xyz, means2D, _rotation, _scaling, _opacity, f_dc, f_rest, face_center, face_orien_mat,
                face_scaling, binding, colors_precomp, raster_settings, grad_sink=None, tanfov=None, rgb8=None,
                float_image=True, depth_alpha=False, hints=None, cameras=None, quantize=N.QUANTIZE_RENDER):
        rs = raster_settings
        ctx.grad_sink = grad_sink
        device = _xyz.device
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
        P, H, W = _xyz.shape[0], int(rs.image_height), int(rs.image_width)
        lead = () if cameras is None else (int(cameras.shape[0]),)
        need_bw = any(ctx.needs_input_grad)
        a = N.ForwardArgs()
        cams = _fill_common(a, rs, device, P, need_bw, cameras)
        a.display_quantize = quantize
        if quantize != N.QUANTIZE_RENDER and (rgb8 is None or need_bw or depth_alpha):
            raise ValueError("the viewer's quantisation writes the display image of a forward-only frame without the "
                             "alpha / depth planes: it needs rgb8=, no gradient and depth_alpha=False")
        binding_orig = binding
        _xyz, _rotation, _scaling, _opacity, f_dc, f_rest, colors_precomp, binding, face_center, face_orien_mat, \
            face_scaling = _fill_bound(a, device, _xyz, _rotation, _scaling, _opacity, f_dc, f_rest, colors_precomp,
                                       binding, face_center, face_orien_mat, face_scaling)
        M, F = a.sh_coeffs, a.num_faces
        tanfov = check_tanfov(tanfov, device)
        rgb8 = check_rgb8(rgb8, rs, device, lead)
        if not float_image and (rgb8 is None or need_bw):
            raise ValueError("float_image=False needs rgb8= and no gradient (the backward reads the float image's state)")
        planes = None
        if depth_alpha:
            planes = (torch.empty(lead + (1, H, W), dtype=torch.float32, device=device),
                      torch.empty(lead + (1, H, W), dtype=torch.float32, device=device))
        color, radii, st, holder = _run_forward(a, device, need_bw, hints, tanfov, rgb8, float_image, planes,
                                                cameras=cameras)
        ctx.tanfov, ctx.cameras = tanfov, cameras
        ctx.depth_alpha = bool(depth_alpha)
        if need_bw:
            ctx.args, ctx.state, ctx.holder = a, st, holder
            ctx.keep = (cams, _xyz, _rotation, _scaling, _opacity, f_dc, f_rest, face_center, face_orien_mat,
                        face_scaling, binding, colors_precomp, radii)
            ctx.dims = (P, M, F)
            ctx.face_shapes = None if binding is None else (face_center.shape, face_orien_mat.shape,
                                                            face_scaling.shape)
            # face-frame gradients are only produced when something upstream of the frame trains (FLAME parameters)
            ctx.want_face = binding is not None and any(ctx.needs_input_grad[7:10])
            ctx.csr = _face_csr(binding_orig, F)[1] if ctx.want_face else None
        ctx.mark_non_differentiable(radii)
        if planes is not None:
            return color, radii, planes[0], planes[1]
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii, *grad_planes):
        a, st = ctx.args, ctx.state
        P, M, F = ctx.dims
        device = ctx.keep[1].device
        binding, colors_precomp = ctx.keep[10], ctx.keep[11]
        g = grad_out_color if grad_out_color.is_contiguous() else grad_out_color.contiguous()
        # frame-sharded data parallel with NVLS: the gradients are reduced INTO the symmetric buffer by the kernel
        flat, symm, (d_xyz, d_rot, d_scale, d_opac, d_dc, d_rest) = _grad_buffer(ctx.grad_sink, P, M, device,
                                                                                 colors_precomp is None)
        use_symm = symm is not None
        # "push": the kernel reduces into every replica with multimem.red; "two_shot": plain stores into the local
        # replica, reduced afterwards by the NVLS all-reduce kernel (dist.SymmetricGradBuffer.end)
        use_mc = use_symm and getattr(symm, "mode", "push") == "push"
        lead = () if ctx.cameras is None else (int(ctx.cameras.shape[0]),)
        d_means2D = torch.empty(lead + (P, 3), dtype=torch.float32, device=device)
        d_colors = torch.empty((P, 3), dtype=torch.float32, device=device) if colors_precomp is not None else None
        d_fc = d_fR = d_fs = None
        if ctx.want_face:
            fshape = ctx.face_shapes
            d_fc = torch.empty(fshape[0], dtype=torch.float32, device=device)
            d_fR = torch.empty(fshape[1], dtype=torch.float32, device=device)
            d_fs = torch.empty(fshape[2], dtype=torch.float32, device=device)
        b = N.BackwardArgs()
        b.abi_version = N.ABI_VERSION
        b.fwd, b.state = C.pointer(a), C.pointer(st)
        b.dL_dout_color = g.data_ptr()
        # parameter-gradient destinations: local addresses, or the same offsets inside the NVLS multicast mapping
        base = (symm.mc_ptr - flat.data_ptr()) if use_mc else 0
        b.grads_are_multicast = int(use_mc)
        b.dL_dmeans3D, b.dL_dopacity = d_xyz.data_ptr() + base, d_opac.data_ptr() + base
        b.dL_dmeans2D = d_means2D.data_ptr()
        b.dL_dcolors = N.ptr(d_colors)
        b.dL_dsh_dc = d_dc.data_ptr() + base
        b.dL_dsh_rest = None if d_rest is None else d_rest.data_ptr() + base
        b.dL_dscales, b.dL_drotations = d_scale.data_ptr() + base, d_rot.data_ptr() + base
        b.dL_dface_center, b.dL_dface_orien_mat, b.dL_dface_scaling = N.ptr(d_fc), N.ptr(d_fR), N.ptr(d_fs)
        if ctx.csr is not None:
            perm, c_face, c_start, c_end = ctx.csr
            b.face_perm, b.face_chunk_face = perm.data_ptr(), c_face.data_ptr()
            b.face_chunk_start, b.face_chunk_end = c_start.data_ptr(), c_end.data_ptr()
            b.num_face_chunks = c_face.shape[0]
        plane_grads = None
        if ctx.depth_alpha:   # gradients of the alpha / depth planes (None: the loss does not read that plane)
            plane_grads = tuple(None if t is None else (t if t.is_contiguous() else t.contiguous()) for t in grad_planes)
        if ctx.cameras is None:
            _run_backward(b, device, ctx.tanfov, plane_grads)
        else:   # the sum over the K views of every single-view gradient but d_means2D, one row per view
            _run_backward(b, device, plane_grads=plane_grads, cameras=ctx.cameras)
        ctx.holder = None
        if ctx.grad_sink is not None:  # dist.py: ONE all-reduce over this buffer instead of six
            ctx.grad_sink.flat_grad = flat
            ctx.grad_sink._gab200_mc_used = bool(use_symm)  # SymmetricGradBuffer.end() only trusts the replica if set
        return (d_xyz, d_means2D, d_rot, d_scale, d_opac, d_dc, d_rest, d_fc, d_fR, d_fs, None, d_colors, None, None,
                None, None, None, None, None, None, None)


def rasterize_bound(raster_settings: GaussianRasterizationSettings, _xyz, _rotation, _scaling, _opacity,
                    features_dc, features_rest, binding=None, face_center=None, face_orien_mat=None,
                    face_scaling=None, means2D=None, colors_precomp=None, grad_sink=None, tanfov=None, rgb8=None,
                    float_image=True, depth_alpha=False, quantize: str = "render"):
    """Fused binding + rasterization.  Returns (color (3,H,W), radii (P,) int32); with depth_alpha=True
    (color, radii, alpha (1,H,W), depth (1,H,W)).

    binding=None is the identity frame (a plain GaussianModel, scene/gaussian_model.py:115-116,127-128,142-143).
    `means2D` is the usual (P,3) gradient holder (its .grad receives dL/dmean2D in NDC units).
    `tanfov`: optional (2,) float32 device tensor {tan(FoVx/2), tan(FoVy/2)} read by the kernels in place of
    raster_settings.tanfovx / tanfovy -- a CUDA graph replay renders whatever was written there before it.  Zero,
    negative or non-finite values cull every splat (image = background).
    `rgb8`: optional contiguous (H,W,3) uint8 CUDA tensor that the forward blend also fills with the display image,
    bit for bit torch's color.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)
    (gab200_forward_display).  float_image=False (rgb8 given, no gradient) skips the float image: color is None.
    quantize="viewer" (rgb8 given, no gradient, no planes): the display bytes are the local viewer's export instead,
    (np.clip(color, 0, 1) * 255).astype(np.uint8) on the float32 image -- no +0.5 (GAB200_QUANTIZE_VIEWER).
    depth_alpha=True (gab200_forward_depth_alpha): also the accumulated alpha 1 - T_final and the alpha-weighted
    view-space depth sum_i w_i z_i (not normalised: depth / alpha is a viewer's depth) of the same blend, both
    differentiable; the colour image, radii and display bytes are those of depth_alpha=False bit for bit.  The gradients
    are plain stores: a grad_sink whose symmetric gradient buffer is in "push" (multicast) mode is refused."""
    if depth_alpha:
        symm = getattr(grad_sink, "symm_grad", None) if grad_sink is not None else None
        if symm is not None and symm.enabled and getattr(symm, "mode", "push") == "push":
            raise ValueError("rasterize_bound(depth_alpha=True) writes plain gradients: use the symmetric gradient "
                             "buffer in 'two_shot' or 'plain' mode, not 'push'")
    if means2D is None:
        means2D = torch.zeros((_xyz.shape[0], 3), dtype=torch.float32, device=_xyz.device)
    if _opacity.ndim == 1:
        _opacity = _opacity[:, None]
    return _RasterizeBound.apply(_xyz, means2D, _rotation, _scaling, _opacity, features_dc, features_rest,
                                 face_center, face_orien_mat, face_scaling, binding, colors_precomp, raster_settings,
                                 grad_sink, tanfov, rgb8, bool(float_image), bool(depth_alpha),
                                 hints_of(grad_sink) if grad_sink is not None else None, None,
                                 N.quantize_mode(quantize))


# ================================================================================================================
# Several cameras of one splat set in one forward (gab200_forward_views)
# ================================================================================================================
def view_hints_of(obj) -> "FrameHints":
    """The FrameHints of a model's multi-view frames, kept apart from its single-view ones (`hints_of`): a K-view
    frame's instance count and depth range are those of K cameras together, and single-view frames must go on
    learning only from single-view frames."""
    h = getattr(obj, "_gab200_view_hints", None)
    if h is None:
        h = FrameHints()
        try:
            obj._gab200_view_hints = h
        except Exception:
            return FrameHints()
    return h


def check_camera_table(cameras, device) -> torch.Tensor:
    """A multi-view camera table: a contiguous (K, 37) float32 tensor on `device`, 1 <= K <= 65535, row k =
    camera_block(cam_k, fov=True)."""
    if not isinstance(cameras, torch.Tensor) or cameras.device != device or cameras.dtype != torch.float32 or \
            cameras.ndim != 2 or cameras.shape[1] != N.CAMERA_FLOATS or not 1 <= cameras.shape[0] <= N.MAX_VIEWS or \
            not cameras.is_contiguous():
        raise ValueError(f"cameras must be a contiguous (K, {N.CAMERA_FLOATS}) float32 tensor on {device} with "
                         f"1 <= K <= {N.MAX_VIEWS} (rows: camera_block(cam, fov=True))")
    return cameras


def rasterize_bound_views(raster_settings: GaussianRasterizationSettings, cameras: torch.Tensor, _xyz, _rotation,
                          _scaling, _opacity, features_dc, features_rest, binding=None, face_center=None,
                          face_orien_mat=None, face_scaling=None, colors_precomp=None, hints: Optional[FrameHints] = None,
                          display: bool = True, float_image: bool = False, depth_alpha: bool = False,
                          quantize: str = "render"):
    """Fused binding + rasterization of K cameras in ONE forward (gab200_forward_views), forward only.

    `cameras`: (K, 37) float32 device table, row k = camera_block(cam_k, fov=True); each view uses its own matrices,
    centre and field of view.  raster_settings gives what the views share: image size, background, scale_modifier,
    sh_degree, debug (its viewmatrix / projmatrix / campos / tanfov* are not read).  Returns (color (K,3,H,W) or None,
    display (K,H,W,3) uint8 or None, radii (K,P) int32, visibility (K,P) bool), every one bit for bit the K
    single-camera forwards' (rasterize_bound(..., rgb8=...)).  `hints`: the capacity / depth hints of these frames
    (view_hints_of(model)); the model's single-view hints are not touched.  No autograd: an input that requires a
    gradient while grad mode is on is refused.
    depth_alpha=True (gab200_forward_views_depth_alpha): also returns alpha and depth, (K,1,H,W) float32 each, the planes
    of rasterize_bound(..., depth_alpha=True) for every view; the other outputs are those of depth_alpha=False bit for
    bit.  quantize: as rasterize_bound's."""
    tensors = [t for t in (_xyz, _rotation, _scaling, _opacity, features_dc, features_rest, face_center,
                           face_orien_mat, face_scaling, colors_precomp) if t is not None]
    if torch.is_grad_enabled() and any(t.requires_grad for t in tensors):
        raise ValueError("rasterize_bound_views is forward only: call it under torch.no_grad() or with detached inputs")
    if not (display or float_image):
        raise ValueError("rasterize_bound_views needs display=True and/or float_image=True")
    rs = raster_settings
    device = _xyz.device
    if device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    cameras = check_camera_table(cameras, device)
    K, H, W = int(cameras.shape[0]), int(rs.image_height), int(rs.image_width)
    rgb8 = torch.empty((K, H, W, 3), dtype=torch.uint8, device=device) if display else None
    if _opacity.ndim == 1:
        _opacity = _opacity[:, None]
    d = lambda t: None if t is None else t.detach()  # noqa: E731  (no gradient: the forward keeps no backward state)
    with torch.no_grad():
        color, radii, *planes = _RasterizeBound.apply(
            d(_xyz), None, d(_rotation), d(_scaling), d(_opacity), d(features_dc), d(features_rest), d(face_center),
            d(face_orien_mat), d(face_scaling), binding, d(colors_precomp), rs, None, None, rgb8, bool(float_image),
            bool(depth_alpha), hints if hints is not None else FrameHints(), cameras, N.quantize_mode(quantize))
    return (color, rgb8, radii, visible_of(radii), *planes)


def rasterize_bound_views_train(raster_settings: GaussianRasterizationSettings, cameras: torch.Tensor, _xyz, _rotation,
                                _scaling, _opacity, features_dc, features_rest, binding=None, face_center=None,
                                face_orien_mat=None, face_scaling=None, means2D=None, colors_precomp=None,
                                grad_sink=None, hints: Optional[FrameHints] = None, depth_alpha: bool = False):
    """Fused binding + rasterization of the K cameras of one timestep as ONE training frame, differentiable.

    `cameras` and `raster_settings` as in rasterize_bound_views.  Returns (color (K,3,H,W), radii (K,P) int32); images
    and radii equal the K single-camera forwards' bit for bit.  The backward writes the sum over the views of every
    single-camera gradient: the raw parameters (into the flat per-splat buffer of rasterize_bound, handed to
    `grad_sink.flat_grad`) and the face frame.  `means2D` is a (K,P,3) holder whose .grad row k receives camera k's
    dL/dmean2D.  `hints`: the capacity / depth hints of these frames (default: view_hints_of(grad_sink)).  The kernels
    exist for SH colours and plain stores only: colors_precomp, and a grad_sink whose symmetric gradient buffer is in
    "push" (multicast) mode, are refused.
    depth_alpha=True (gab200_forward_views_train_depth_alpha / gab200_backward_views_depth_alpha): returns (color,
    radii, alpha (K,1,H,W), depth (K,1,H,W)), each view's planes those of rasterize_bound(..., depth_alpha=True),
    differentiable in all three images; the backward writes the sum over the views of the single-camera gradients of
    the whole loss (a mask or depth term included)."""
    if colors_precomp is not None:
        raise ValueError("rasterize_bound_views_train takes SH colours only (no colors_precomp)")
    symm = getattr(grad_sink, "symm_grad", None) if grad_sink is not None else None
    if symm is not None and symm.enabled and getattr(symm, "mode", "push") == "push":
        raise ValueError("rasterize_bound_views_train writes plain gradients: use the symmetric gradient buffer in "
                         "'two_shot' or 'plain' mode, not 'push'")
    device = _xyz.device
    if device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    cameras = check_camera_table(cameras, device)
    K, P = int(cameras.shape[0]), int(_xyz.shape[0])
    if means2D is None:
        means2D = torch.zeros((K, P, 3), dtype=torch.float32, device=device)
    elif tuple(means2D.shape) != (K, P, 3):
        raise ValueError(f"means2D must be a ({K}, {P}, 3) holder, got {tuple(means2D.shape)}")
    if _opacity.ndim == 1:
        _opacity = _opacity[:, None]
    if hints is None:
        hints = view_hints_of(grad_sink) if grad_sink is not None else FrameHints()
    return _RasterizeBound.apply(_xyz, means2D, _rotation, _scaling, _opacity, features_dc, features_rest, face_center,
                                 face_orien_mat, face_scaling, binding, None, raster_settings, grad_sink, None, None,
                                 True, bool(depth_alpha), hints, cameras)


def bind_activate(raster_settings_or_modifier, _xyz, _rotation, _scaling, _opacity, binding=None, face_center=None,
                  face_orien_mat=None, face_scaling=None):
    """Exports what the fused preprocess computes for the binding (no autograd): world means3D (P,3), opacities (P,1),
    scales (P,3), cov3D (P,6).  Same device code as the fused forward -> bit-identical values."""
    device = _xyz.device
    P = _xyz.shape[0]
    mod = raster_settings_or_modifier.scale_modifier if isinstance(raster_settings_or_modifier, tuple) \
        else float(raster_settings_or_modifier)
    a = N.ForwardArgs()
    a.abi_version, a.input_mode, a.P, a.scale_modifier = N.ABI_VERSION, N.INPUT_BOUND_RAW, P, mod
    keep = [_f32c(_xyz.detach(), "_xyz", device), _f32c(_rotation.detach(), "_rotation", device),
            _f32c(_scaling.detach(), "_scaling", device), _f32c(_opacity.detach(), "_opacity", device)]
    a.means3D, a.rotations, a.scales, a.opacities = (t.data_ptr() for t in keep)
    if binding is not None:
        keep += [binding.to(torch.int32).contiguous(), _f32c(face_center.detach(), "face_center", device),
                 _f32c(face_orien_mat.detach(), "face_orien_mat", device),
                 _f32c(face_scaling.detach(), "face_scaling", device)]
        a.binding, a.face_center, a.face_orien_mat, a.face_scaling = (t.data_ptr() for t in keep[4:])
        a.num_faces = keep[5].shape[0]
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=device)  # noqa: E731
    means3D, opac, scales, cov = e(P, 3), e(P, 1), e(P, 3), e(P, 6)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        N.check(N.lib().gab200_bind_activate(C.byref(a), means3D.data_ptr(), opac.data_ptr(), scales.data_ptr(),
                                             cov.data_ptr(), C.c_void_p(stream)), "gab200_bind_activate")
    return means3D, opac, scales, cov


# ================================================================================================================
# Per-face frame (SURVEY.md 8f rank 1): one launch instead of ~25 eager ones, differentiable w.r.t. the vertices
# ================================================================================================================
class _FaceFrame(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces):
        device = verts.device
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
        v = _f32c(verts.reshape(-1, 3), "verts", device)
        f = faces if faces.dtype == torch.int32 else faces.to(torch.int32)
        f = f.contiguous()
        V, F = v.shape[0], f.shape[0]
        fc = torch.empty((F, 3), dtype=torch.float32, device=device)
        fR = torch.empty((F, 3, 3), dtype=torch.float32, device=device)
        fs = torch.empty((F, 1), dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_face_frame_forward(F, V, v.data_ptr(), f.data_ptr(), fc.data_ptr(), fR.data_ptr(),
                                                      fs.data_ptr(), C.c_void_p(stream)), "gab200_face_frame_forward")
        ctx.keep = (v, f, verts.shape)
        return fc, fR, fs

    @staticmethod
    def backward(ctx, g_fc, g_fR, g_fs):
        v, f, shape = ctx.keep
        device = v.device
        gv = torch.empty_like(v)
        c = lambda t: None if t is None else (t if t.is_contiguous() else t.contiguous())  # noqa: E731
        g_fc, g_fR, g_fs = c(g_fc), c(g_fR), c(g_fs)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_face_frame_backward(f.shape[0], v.shape[0], v.data_ptr(), f.data_ptr(), N.ptr(g_fc),
                                                       N.ptr(g_fR), N.ptr(g_fs), gv.data_ptr(), C.c_void_p(stream)),
                    "gab200_face_frame_backward")
        return gv.view(shape), None


def face_frame(verts: torch.Tensor, faces: torch.Tensor):
    """verts (V,3) [or (1,V,3)], faces (F,3) -> face_center (F,3), face_orien_mat (F,3,3), face_scaling (F,1).
    Replaces update_mesh_properties / compute_face_orientation (scene/flame_gaussian_model.py:137-147)."""
    return _FaceFrame.apply(verts, faces)


# ================================================================================================================
# L1 loss against a uint8 ground truth (SURVEY.md 8f rank 2): loss and dL/dimage in one kernel
# ================================================================================================================
class _L1LossU8(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt_u8):
        device = image.device
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
        img = _f32c(image, "image", device)
        if gt_u8.dtype != torch.uint8 or gt_u8.numel() != img.numel():
            raise TypeError("gt must be a uint8 tensor with the image's number of elements")
        gt = gt_u8 if gt_u8.is_contiguous() else gt_u8.contiguous()
        loss = torch.empty((), dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_l1_loss_u8(img.numel(), img.data_ptr(), gt.data_ptr(), None, loss.data_ptr(),
                                              C.c_void_p(stream)), "gab200_l1_loss_u8")
        ctx.save_for_backward(img, gt)
        return loss

    @staticmethod
    def backward(ctx, g):
        img, gt = ctx.saved_tensors
        device = img.device
        grad = torch.empty_like(img)
        gs = g if (g.dtype == torch.float32 and g.device == device) else g.to(device=device, dtype=torch.float32)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_l1_loss_u8_backward(img.numel(), img.data_ptr(), gt.data_ptr(), gs.data_ptr(),
                                                       grad.data_ptr(), C.c_void_p(stream)), "gab200_l1_loss_u8_backward")
        return grad, None


def l1_loss_u8(image: torch.Tensor, gt_u8: torch.Tensor) -> torch.Tensor:
    """mean |image - gt/255| for a uint8 ground truth (same shape), differentiable w.r.t. `image`."""
    return _L1LossU8.apply(image, gt_u8)
