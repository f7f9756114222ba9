"""The two callers either side of the rasterizer in the reference's training step (SURVEY.md 8f ranks 2 and 3), as
CUDA launches behind the same C ABI:

  photometric_loss(image, gt, lambda_dssim)   <- l1_loss * (1 - lambda) + (1 - ssim) * lambda
                                                 (utils/loss_utils.py:17-18,36-63, train.py:131-132)
  composite_rgba(rgba_u8, bg, size=None)      <- the loader's RGBA composite onto the background, and the alpha
                                                 mask it drops (scene/__init__.py:48-51); with `size`, then its
                                                 resize to the camera's size (PILtoTorch, resize.py)
  image_metrics(render, gt_u8)                <- clamp + l1_loss, psnr, ssim of one val / test view (train.py:277-288)
                                                 and metrics.py:71-74 (evaluation, forward only)
  Adam(param_groups, lr, betas, eps)          <- torch.optim.Adam(l, lr=0.0, eps=1e-15).step()
                                                 (scene/gaussian_model.py:213-232, train.py:207-210)
  Adam(..., capturable=True)                  <- the same step with the step counters, the bias corrections and the
     + expon_lr_schedule(...)                    xyz learning-rate schedule (update_learning_rate, train.py:106) on
                                                 the device: capturable into a CUDA graph

No CPU or eager fallback: each raises when the library is missing or a tensor is not a CUDA tensor of the right dtype.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _native as N
from .resize import check_size, resize_u8


# ================================================================================================================
# (1 - lambda) L1 + lambda (1 - SSIM), loss and dL/dimage in two launches
# ================================================================================================================
class _PhotometricLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, lambda_dssim):
        device = image.device
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
        if image.dtype != torch.float32 or image.dim() not in (3, 4):
            raise TypeError("image must be a float32 (C, H, W) or (B, C, H, W) tensor")
        if gt.shape != image.shape or gt.device != device:
            raise ValueError(f"gt must have the image's shape {tuple(image.shape)} on {device}, got {tuple(gt.shape)} on {gt.device}")
        if gt.dtype not in (torch.uint8, torch.float32):
            raise TypeError(f"gt must be uint8 (value/255) or float32, got {gt.dtype}")
        if not 0.0 <= float(lambda_dssim) <= 1.0:
            raise ValueError("lambda_dssim must lie in [0, 1]")
        img = image if image.is_contiguous() else image.contiguous()
        g = gt if gt.is_contiguous() else gt.contiguous()
        H, W = int(img.shape[-2]), int(img.shape[-1])
        Cc = img.numel() // max(H * W, 1)   # a batch is just more independent planes: the means run over all of them
        grad = torch.empty_like(img)
        scratch = torch.empty(N.PHOTOMETRIC_SCRATCH_HEAD + 3 * img.numel(), dtype=torch.float32, device=device)
        loss = torch.empty(3, dtype=torch.float32, device=device)
        a = N.PhotometricArgs()
        a.abi_version = N.ABI_VERSION
        a.channels, a.height, a.width = Cc, H, W
        a.gt_is_u8 = 1 if gt.dtype == torch.uint8 else 0
        a.lambda_dssim = float(lambda_dssim)
        a.image, a.gt, a.grad = img.data_ptr(), g.data_ptr(), grad.data_ptr()
        a.loss, a.scratch = loss.data_ptr(), scratch.data_ptr()
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_photometric_loss(C.byref(a), C.c_void_p(stream)), "gab200_photometric_loss")
        ctx.save_for_backward(grad)
        ctx.mark_non_differentiable(loss)
        return loss[2], loss

    @staticmethod
    def backward(ctx, g_total, _g_parts):
        (grad,) = ctx.saved_tensors
        return grad.mul_(g_total), None, None  # in place: the buffer is ours and single-use


def photometric_loss(image: torch.Tensor, gt: torch.Tensor, lambda_dssim: float = 0.2, return_parts: bool = False):
    """`(1 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1 - ssim(image, gt))` of the reference training
    loop, differentiable w.r.t. `image` (float32, (C, H, W) or (B, C, H, W) like the reference's `ssim`).  `gt` is float32 in [0, 1] like `viewpoint_cam.original_image`
    or the uint8 image it was decoded from (value/255 in-kernel: a quarter of the upload).  With `return_parts` also
    returns the detached tensor [l1 mean, ssim mean, total] (for logging, train.py:159-166)."""
    total, parts = _PhotometricLoss.apply(image, gt, lambda_dssim)
    return (total, parts) if return_parts else total


# ================================================================================================================
# The loader's RGBA composite: a capture's decoded RGBA frames -> the uint8 ground truth and the alpha mask, one launch
# ================================================================================================================
def check_rgba(rgba_u8: torch.Tensor) -> int:
    """The checks of composite_rgba; returns the number of frames (1 for an (H,W,4) frame)."""
    if not isinstance(rgba_u8, torch.Tensor) or rgba_u8.dtype != torch.uint8 or rgba_u8.dim() not in (3, 4) or \
            rgba_u8.shape[-1] != 4:
        raise TypeError("rgba must be a uint8 (H, W, 4) or (K, H, W, 4) tensor, got "
                        f"{getattr(rgba_u8, 'dtype', type(rgba_u8))} {tuple(getattr(rgba_u8, 'shape', ()))}")
    if rgba_u8.device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    return 1 if rgba_u8.dim() == 3 else int(rgba_u8.shape[0])


def launch_composite_rgba(rgba_u8: torch.Tensor, bg: torch.Tensor, gt_out: torch.Tensor,
                          mask_out: Optional[torch.Tensor] = None):
    """Enqueues gab200_composite_rgba on the current stream: rgba (H,W,4) / (K,H,W,4) uint8 -> gt_out (3,H,W) /
    (K,3,H,W) uint8 and mask_out (1,H,W) / (K,1,H,W) uint8 (None: not written).  bg: 3 float32 on the device, read by
    the kernel.  Capturable: it reads nothing on the host."""
    views = check_rgba(rgba_u8)
    device = rgba_u8.device
    H, W = int(rgba_u8.shape[-3]), int(rgba_u8.shape[-2])
    lead = () if rgba_u8.dim() == 3 else (views,)
    for t, n, c in ((gt_out, "gt_out", 3), (mask_out, "mask_out", 1)):
        if t is not None and (t.dtype != torch.uint8 or tuple(t.shape) != lead + (c, H, W) or t.device != device
                              or not t.is_contiguous()):
            raise ValueError(f"{n} must be a contiguous uint8 {lead + (c, H, W)} tensor on {device}")
    if bg.dtype != torch.float32 or bg.numel() != 3 or bg.device != device or not bg.is_contiguous():
        raise ValueError(f"bg must be 3 contiguous float32 values on {device}")
    src = rgba_u8 if rgba_u8.is_contiguous() else rgba_u8.contiguous()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        N.check(N.lib().gab200_composite_rgba(views, H, W, src.data_ptr(), bg.data_ptr(), gt_out.data_ptr(),
                                              N.ptr(mask_out), C.c_void_p(stream)), "gab200_composite_rgba")
    return gt_out, mask_out


@torch.no_grad()
def composite_rgba(rgba_u8: torch.Tensor, bg, size=None) -> tuple:
    """(gt_u8, mask_u8) of decoded RGBA capture frames, computed on the device: what the reference's loader
    (CameraDataset.__getitem__, scene/__init__.py:48-51) makes of `np.array(Image.open(p).convert("RGBA"))` on the
    host, bit for bit, plus the alpha channel it throws away.

    rgba_u8: a CUDA uint8 (H, W, 4) frame or (K, H, W, 4) frames.  bg: the camera's background (3 values, 0 or 1 per
    channel in the reference; other colours go through the same formula).  Returns the uint8 ground truth (3, H, W) /
    (K, 3, H, W) -- trunc((c/255 * a/255 + bg * (1 - a/255)) * 255) in float64, the loader's bytes -- and the alpha
    bytes (1, H, W) / (K, 1, H, W), the foreground mask (value/255) of a mask loss.

    size (width, height): the frames are composited at their own size, then resized to it as the loader's PILtoTorch
    resizes them (resize.resize_u8: PIL's bicubic resize of the "RGB" image, bit for bit) -- the ground truth of a
    camera whose size differs from its files' (resize.loader_size).  The mask is resized as PIL resizes an "L" image
    of the alpha bytes; the reference drops alpha, so that resized mask is this project's definition.  Capturable."""
    if size is not None:
        width, height = check_size(size)
        gt, mask = composite_rgba(rgba_u8, bg)
        if (width, height) == (int(gt.shape[-1]), int(gt.shape[-2])):
            return gt, mask   # PIL's resize to the image's own size is a copy
        return resize_u8(gt, width, height), resize_u8(mask, width, height)
    views = check_rgba(rgba_u8)
    device = rgba_u8.device
    H, W = int(rgba_u8.shape[-3]), int(rgba_u8.shape[-2])
    lead = () if rgba_u8.dim() == 3 else (views,)
    b = torch.as_tensor(bg, dtype=torch.float32).reshape(-1).to(device).contiguous()
    if b.numel() != 3:
        raise ValueError(f"bg must hold 3 values, got {b.numel()}")
    gt = torch.empty(lead + (3, H, W), dtype=torch.uint8, device=device)
    mask = torch.empty(lead + (1, H, W), dtype=torch.uint8, device=device)
    return launch_composite_rgba(rgba_u8, b, gt, mask)


# ================================================================================================================
# Evaluation metrics: l1, psnr (two definitions) and ssim of one view, forward only, in two launches
# ================================================================================================================
METRIC_NAMES = ("l1", "psnr", "psnr_all", "ssim")


def check_metrics_inputs(render: torch.Tensor, gt_u8: torch.Tensor) -> int:
    """The checks of image_metrics; returns the render kind (_native.METRICS_FLOAT_CHW or METRICS_U8_HWC)."""
    device = render.device
    if render.dtype == torch.float32 and render.dim() == 3 and render.shape[0] == 3:
        kind, H, W = N.METRICS_FLOAT_CHW, int(render.shape[1]), int(render.shape[2])
    elif render.dtype == torch.uint8 and render.dim() == 3 and render.shape[2] == 3:
        kind, H, W = N.METRICS_U8_HWC, int(render.shape[0]), int(render.shape[1])
    else:
        raise TypeError("render must be a float32 (3, H, W) image or the uint8 (H, W, 3) display image, got "
                        f"{render.dtype} {tuple(render.shape)}")
    if gt_u8.dtype != torch.uint8:
        raise TypeError(f"gt_u8 must be uint8 (value/255), got {gt_u8.dtype}")
    if tuple(gt_u8.shape) != (3, H, W) or gt_u8.device != device:
        raise ValueError(f"gt_u8 must have shape (3, {H}, {W}) on {device}, got {tuple(gt_u8.shape)} on {gt_u8.device}")
    if H == 0 or W == 0:
        raise ValueError("an empty image has no metrics")
    if device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    return kind


def metrics_scratch(height: int, width: int, device) -> torch.Tensor:
    """Device scratch for one gab200_image_metrics call of this size (the per-tile partial sums)."""
    nbytes = int(N.lib().gab200_image_metrics_scratch_bytes(int(height), int(width)))
    return torch.empty(max(nbytes, 8), dtype=torch.uint8, device=device)


def launch_image_metrics(render: torch.Tensor, gt_u8: torch.Tensor, table: torch.Tensor,
                         row: Optional[torch.Tensor] = None, skip_flag: Optional[torch.Tensor] = None,
                         scratch: Optional[torch.Tensor] = None):
    """Enqueues the metrics of `render` against `gt_u8` into row `*row` (a device int32; None = row 0) of `table`, a
    (rows, 4) float32 device tensor, on the current stream; nothing is written when `skip_flag` (device int32) holds a
    non-zero value as the kernel runs.  Capturable: it reads nothing on the host."""
    kind = check_metrics_inputs(render, gt_u8)
    device = render.device
    if table.dtype != torch.float32 or table.dim() != 2 or table.shape[1] != N.METRICS_FIELDS or \
            table.device != device or not table.is_contiguous() or table.shape[0] < 1:
        raise ValueError(f"table must be a contiguous float32 (rows, {N.METRICS_FIELDS}) tensor on {device}")
    for t, n in ((row, "row"), (skip_flag, "skip_flag")):
        if t is not None and (t.dtype != torch.int32 or t.device != device):
            raise TypeError(f"{n} must be an int32 tensor on {device}")
    r = render if render.is_contiguous() else render.contiguous()
    g = gt_u8 if gt_u8.is_contiguous() else gt_u8.contiguous()
    H, W = (int(r.shape[1]), int(r.shape[2])) if kind == N.METRICS_FLOAT_CHW else (int(r.shape[0]), int(r.shape[1]))
    if scratch is None:
        scratch = metrics_scratch(H, W, device)
    elif scratch.numel() * scratch.element_size() < int(N.lib().gab200_image_metrics_scratch_bytes(H, W)):
        raise ValueError("metrics scratch too small for this image size")
    a = N.MetricsArgs()
    a.abi_version, a.height, a.width, a.render_kind = N.ABI_VERSION, H, W, kind
    a.render, a.gt, a.row, a.table = r.data_ptr(), g.data_ptr(), N.ptr(row), table.data_ptr()
    a.table_rows, a.skip_flag, a.scratch = int(table.shape[0]), N.ptr(skip_flag), scratch.data_ptr()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        N.check(N.lib().gab200_image_metrics(C.byref(a), C.c_void_p(stream)), "gab200_image_metrics")
    return table


@torch.no_grad()
def image_metrics(render: torch.Tensor, gt_u8: torch.Tensor) -> torch.Tensor:
    """(4,) float32 device tensor {l1, psnr, psnr_all, ssim} of one view (include/gab200_rasterizer.h,
    gab200_image_metrics), with no autograd and no host wait.

    render: the float32 (3, H, W) image of render(), clamped to [0, 1] in the kernel as training_report clamps it
    (train.py:277), or the uint8 (H, W, 3) display image of render_display() -- the bytes render.py writes as a PNG,
    read back as value/255 as metrics.py reads them.  gt_u8: the uint8 (3, H, W) ground truth (value/255).
      l1       = l1_loss(image, gt)                                  (train.py:286)
      psnr     = psnr(image, gt).mean(): one PSNR per channel, averaged (train.py:287 passes a [3,H,W] image)
      psnr_all = psnr over all values at once (metrics.py:73 passes [1,3,H,W] tensors)
      ssim     = ssim(image, gt)                                     (train.py:288, metrics.py:72)
    Sums run in double with a fixed reduction order: two calls on the same inputs give the same bits."""
    table = torch.empty((1, N.METRICS_FIELDS), dtype=torch.float32, device=render.device)
    return launch_image_metrics(render, gt_u8, table)[0]


# ================================================================================================================
# Adam: all parameter groups in one launch
# ================================================================================================================
def expon_lr_schedule(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000) -> dict:
    """The reference's `get_expon_lr_func(lr_init, lr_final, lr_delay_steps, lr_delay_mult, max_steps)`
    (utils/general_utils.py) as a parameter group's `"lr_schedule"` for a capturable `Adam`, which evaluates it on the
    device at every step.  The reference's `xyz` schedule (scene/gaussian_model.py:224-227) is
    `expon_lr_schedule(lr_init=position_lr_init * spatial_lr_scale, lr_final=position_lr_final * spatial_lr_scale,
    lr_delay_mult=position_lr_delay_mult, max_steps=position_lr_max_steps)`."""
    sched = dict(lr_init=float(lr_init), lr_final=float(lr_final), lr_delay_steps=int(lr_delay_steps),
                 lr_delay_mult=float(lr_delay_mult), max_steps=int(max_steps))
    if sched["lr_init"] < 0 or sched["lr_final"] < 0 or sched["lr_delay_steps"] < 0 or sched["lr_delay_mult"] < 0 \
            or sched["max_steps"] <= 0:
        raise ValueError(f"invalid learning-rate schedule {sched}")
    return sched


class Adam(torch.optim.Optimizer):
    """Drop-in for `torch.optim.Adam(param_groups, lr=0.0, eps=1e-15)` as the reference builds it.

    Same `param_groups` / `state` layout as torch's Adam (`state[p] = {"step", "exp_avg", "exp_avg_sq"}`), so the
    reference's densification surgery on the optimizer state (scene/gaussian_model.py:334-419) and
    `optimizer.state_dict()` checkpoints (scene/gaussian_model.py:89,111) work unchanged.  amsgrad, weight decay and
    maximize are not part of the reference's configuration and are rejected.

    capturable=True: torch's layout for `capturable=True` -- `state["step"]` is a float32 scalar on the parameter's
    device -- and `step()` reads nothing on the host, so it can be captured into a CUDA graph (graph.GraphedFrame) and
    replayed.  The step counters are incremented and the bias corrections formed on the device
    (gab200_adam_step_device).  A group may then carry `"lr_schedule": expon_lr_schedule(...)`: its learning rate is
    the reference's exponential schedule at the group's new step, which in train.py equals `iteration`, so
    `update_learning_rate(iteration)` is no longer needed for it.  A constant `lr` written into a group between
    replays is NOT seen by a captured step (it was baked in at capture).  Create the state before a capture
    (`init_state()`): state created inside one would be re-zeroed by every replay."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, maximize=False,
                 capturable=False):
        if weight_decay != 0 or amsgrad or maximize:
            raise ValueError("gaussianavatars_b200.Adam implements the reference configuration only "
                             "(weight_decay=0, amsgrad=False, maximize=False)")
        if not 0.0 <= lr or not 0.0 <= eps or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("invalid Adam hyper-parameters")
        # weight_decay is the one key torch.optim.Adam reads from a loaded group without filling in a default: with it
        # a checkpoint of this optimizer loads into torch's Adam and steps there
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=0.0, capturable=bool(capturable)))

    def _new_state(self, p, capturable):
        st = self.state[p]
        if capturable:
            st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
        else:
            st["step"] = torch.tensor(0.0, dtype=torch.float32)
        st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    @torch.no_grad()
    def init_state(self):
        """Creates the state (step 0, zero moments) of every parameter of a capturable group that has none yet --
        what the first eager step() would create, which makes no step itself."""
        for group in self.param_groups:
            if group.get("capturable", False):
                for p in group["params"]:
                    if len(self.state[p]) == 0:
                        self._new_state(p, True)

    @torch.no_grad()
    def step(self, closure=None, skip_flag: Optional[torch.Tensor] = None):
        """skip_flag (capturable groups only): an int32 device tensor; when it holds a non-zero value as the step
        executes, the step changes no parameter, moment or step counter (graph.GraphedFrame passes its sticky
        instance-overflow flag)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        batches = {}   # (device, step, beta1, beta2, eps) -> list of segments; one launch per 8 segments
        device_batches = {}   # capturable groups: (device, beta1, beta2, eps) -> list of segments
        keep = []
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            capturable = group.get("capturable", False)
            sched = group.get("lr_schedule")
            if sched is not None and not capturable:
                raise ValueError("a group's lr_schedule is evaluated on the device: it needs Adam(capturable=True)")
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.device.type != "cuda" or p.dtype != torch.float32 or p.grad.is_sparse or not p.is_contiguous():
                    raise RuntimeError("gaussianavatars_b200.Adam steps contiguous CUDA float32 parameters only "
                                       "(no CPU or eager fallback)")
                st = self.state[p]
                if len(st) == 0:
                    if capturable and torch.cuda.is_current_stream_capturing():
                        raise RuntimeError("capturable Adam: call init_state() before capturing step()")
                    st = self._new_state(p, capturable)
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                m, v = st["exp_avg"], st["exp_avg_sq"]
                if not (m.is_contiguous() and v.is_contiguous()):
                    raise RuntimeError("Adam state tensors must be contiguous")
                keep.append(g)
                if capturable:
                    t = st["step"]
                    if t.device != p.device or t.dtype != torch.float32 or t.numel() != 1:
                        raise RuntimeError("capturable Adam keeps state['step'] as a float32 scalar on the "
                                           "parameter's device")
                    seg = N.AdamDeviceSegment(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                              t.data_ptr(), float(group["lr"]))
                    if sched is not None:
                        seg.has_schedule = 1
                        seg.lr_init, seg.lr_final = float(sched["lr_init"]), float(sched["lr_final"])
                        seg.lr_delay_mult = float(sched.get("lr_delay_mult", 1.0))
                        seg.lr_delay_steps = int(sched.get("lr_delay_steps", 0))
                        seg.max_steps = int(sched["max_steps"])
                    key = (p.device, float(beta1), float(beta2), float(group["eps"]))
                    device_batches.setdefault(key, []).append(seg)
                    continue
                st["step"] += 1
                seg = N.AdamSegment(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), float(group["lr"]))
                key = (p.device, int(st["step"]), float(beta1), float(beta2), float(group["eps"]))
                batches.setdefault(key, []).append(seg)
        for (device, step, beta1, beta2, eps), segs in batches.items():
            arr = (N.AdamSegment * len(segs))(*segs)
            with torch.cuda.device(device):
                stream = torch.cuda.current_stream(device).cuda_stream
                N.check(N.lib().gab200_adam_step(len(segs), arr, step, beta1, beta2, eps, C.c_void_p(stream)),
                        "gab200_adam_step")
        for (device, beta1, beta2, eps), segs in device_batches.items():
            arr = (N.AdamDeviceSegment * len(segs))(*segs)
            flag = None
            if skip_flag is not None:
                if skip_flag.device != device or skip_flag.dtype != torch.int32:
                    raise TypeError(f"skip_flag must be an int32 tensor on {device}")
                flag = skip_flag.data_ptr()
            with torch.cuda.device(device):
                stream = torch.cuda.current_stream(device).cuda_stream
                N.check(N.lib().gab200_adam_step_device(len(segs), arr, beta1, beta2, eps, flag, C.c_void_p(stream)),
                        "gab200_adam_step_device")
        return loss


# ================================================================================================================
# position / scale regularisers of the mesh-bound training step (train.py:134-146), loss + gradient in one launch each
# ================================================================================================================
class _BindingRegularizers(torch.autograd.Function):
    @staticmethod
    def forward(ctx, _xyz, _scaling, face_scaling, radii, binding, thr_xyz, thr_scale, lam_xyz, lam_scale, metric_xyz,
                metric_scale):
        device = _xyz.device
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
        for t, n in ((_xyz, "_xyz"), (_scaling, "_scaling")):
            if t.dtype != torch.float32 or t.shape != (_xyz.shape[0], 3):
                raise TypeError(f"{n} must be a float32 (P, 3) tensor")
        P = _xyz.shape[0]
        x = _xyz if _xyz.is_contiguous() else _xyz.contiguous()
        s = _scaling if _scaling.is_contiguous() else _scaling.contiguous()
        r = radii if radii.dtype == torch.int32 else radii.to(torch.int32)   # a bool visibility_filter works as well
        r = r if r.is_contiguous() else r.contiguous()
        if r.numel() != P:
            raise ValueError("radii / visibility_filter must have one entry per splat")
        a = N.RegularizeArgs()
        a.abi_version, a.P = N.ABI_VERSION, P
        a.metric_xyz, a.metric_scale = int(bool(metric_xyz)), int(bool(metric_scale))
        a.threshold_xyz, a.threshold_scale = float(thr_xyz), float(thr_scale)
        a.lambda_xyz, a.lambda_scale = float(lam_xyz), float(lam_scale)
        a.xyz, a.scaling, a.radii = x.data_ptr(), s.data_ptr(), r.data_ptr()
        keep = [x, s, r]
        if binding is not None:
            b = binding if binding.dtype == torch.int32 else binding.to(torch.int32)
            fs = face_scaling.reshape(-1)
            fs = fs if fs.is_contiguous() else fs.contiguous()
            a.binding, a.face_scaling = b.data_ptr(), fs.data_ptr()
            keep += [b, fs]
        loss = torch.empty(3, dtype=torch.float32, device=device)
        sums = torch.empty(3, dtype=torch.float64, device=device)
        a.loss, a.sums = loss.data_ptr(), sums.data_ptr()
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_regularize_forward(C.byref(a), C.c_void_p(stream)), "gab200_regularize_forward")
        ctx.args, ctx.keep, ctx.sums = a, keep, sums
        ctx.face_shape = None if face_scaling is None else face_scaling.shape
        ctx.want_face = binding is not None and face_scaling is not None and ctx.needs_input_grad[2] and \
            (metric_xyz or metric_scale)
        ctx.mark_non_differentiable(loss)
        return loss[0], loss[1], loss

    @staticmethod
    def backward(ctx, g_xyz, g_scale, _g_all):
        a = ctx.args
        device = ctx.keep[0].device
        P = a.P
        gx = torch.empty((P, 3), dtype=torch.float32, device=device)
        gs = torch.empty((P, 3), dtype=torch.float32, device=device)
        gf = torch.zeros(ctx.face_shape, dtype=torch.float32, device=device) if ctx.want_face else None
        z = torch.zeros((), dtype=torch.float32, device=device)
        g = torch.stack((g_xyz if g_xyz is not None else z, g_scale if g_scale is not None else z)).float().contiguous()
        a.grad_xyz, a.grad_scaling, a.grad_face_scaling = gx.data_ptr(), gs.data_ptr(), N.ptr(gf)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(N.lib().gab200_regularize_backward(C.byref(a), g.data_ptr(), C.c_void_p(stream)),
                    "gab200_regularize_backward")
        return gx, gs, gf, None, None, None, None, None, None, None, None


def binding_regularizers(_xyz, _scaling, radii, binding=None, face_scaling=None, threshold_xyz=1.0, threshold_scale=0.6,
                         lambda_xyz=1e-2, lambda_scale=1.0, metric_xyz=False, metric_scale=False, return_count=False):
    """`losses['xyz']`, `losses['scale']` of the reference training step (train.py:134-146; defaults
    arguments/__init__.py:100-105), differentiable w.r.t. `_xyz`, `_scaling` (and `face_scaling` in the metric
    variants).  `radii` is the rendered frame's radii (or its `visibility_filter`).  A training step that adds these
    two to the photometric loss never calls `get_scaling` / boolean-mask indexing."""
    lx, ls, all_ = _BindingRegularizers.apply(_xyz, _scaling, face_scaling, radii, binding, threshold_xyz, threshold_scale,
                                              lambda_xyz, lambda_scale, metric_xyz, metric_scale)
    return (lx, ls, all_[2]) if return_count else (lx, ls)
