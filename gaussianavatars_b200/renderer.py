"""Drop-in for gaussian_renderer.render() (reference: gaussian_renderer/__init__.py:19-101).

`render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, override_color=None)` returns the same dict
{"render", "viewspace_points", "visibility_filter", "radii"}.  Two routes:

  * reference route  -- pc's getters (get_xyz / get_scaling / ...) feed `GaussianRasterizer` exactly as the
    reference does (also taken when pipe.compute_cov3D_python or pipe.convert_SHs_python is set);
  * fused route      -- when `pc` exposes the raw parameters (`_xyz, _rotation, _scaling, _opacity, _features_dc,
    _features_rest`) the binding of scene/gaussian_model.py:113-160 runs inside the preprocess kernel
    (`rasterize_bound`): no getter, no torch.cat, no (P,3,3) temporaries, one flat gradient buffer.
Camera matrices that live on the host are uploaded once and cached on the camera object (the reference re-uploads
three tensors per call, gaussian_renderer/__init__.py:44-47).
A camera may carry its field of view in device memory as `cam.tanfov`, a (2,) float32 CUDA tensor
{tan(FoVx/2), tan(FoVy/2)} (graph.GraphedFrame(per_camera_fov=True) does): the fused route's kernels read it there
instead of FoVx / FoVy; the reference route cannot and refuses such a camera.
`render_views(cameras, ...)` renders every camera of a rig (one image size) in one forward, forward only;
`render_views_train(cameras, ...)` is its differentiable form, for a training step over every camera of a timestep.
`depth_alpha=True` (render, render_bound, render_display; fused route only) adds "alpha" (1,H,W), the accumulated
opacity 1 - T_final, and "depth" (1,H,W), the alpha-weighted view-space depth, both from the colour blend itself;
on render_views and render_views_train it adds them for every camera, (K,1,H,W).
"""
from __future__ import annotations

import math

import torch

from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, check_camera_table, hints_of,
                         rasterize_bound, rasterize_bound_views, rasterize_bound_views_train, view_hints_of,
                         visible_of)


def _camera_block(cam, device):
    cached = getattr(cam, "_gab200_dev", None)
    if cached is not None and cached[0] == device and cached[1] is cam.world_view_transform:
        return cached[2]
    blk = (cam.world_view_transform.to(device=device, dtype=torch.float32).contiguous(),
           cam.full_proj_transform.to(device=device, dtype=torch.float32).contiguous(),
           cam.camera_center.to(device=device, dtype=torch.float32).contiguous())
    try:
        cam._gab200_dev = (device, cam.world_view_transform, blk)
    except Exception:  # read-only camera objects: just do not cache
        pass
    return blk


def _settings(cam, pc, pipe, bg_color, scaling_modifier, device, size=None):
    """The settings of a frame of camera object `cam`, or of a (K, 37) camera table `cam` of image `size` (W, H): the
    views' matrices, centres and fields of view are then in the table, and the settings carry none."""
    if size is None:
        W, H = int(cam.image_width), int(cam.image_height)
        view, proj, center = _camera_block(cam, device)
        tanfovx, tanfovy = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    else:
        (W, H), view, proj, center, tanfovx, tanfovy = size, None, None, None, 1.0, 1.0
    return GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=tanfovx, tanfovy=tanfovy, bg=bg_color,
        scale_modifier=scaling_modifier, viewmatrix=view, projmatrix=proj, sh_degree=pc.active_sh_degree,
        campos=center, prefiltered=False, debug=bool(getattr(pipe, "debug", False)))


def _has_raw(pc):
    return all(hasattr(pc, n) for n in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest"))


def _fused_frame(cam, pc, pipe, bg_color, scaling_modifier, size=None):
    """The settings of a fused-route frame (of a camera, or of a camera table of image `size`), the binding and the
    model's face frame (None without a binding)."""
    rs = _settings(cam, pc, pipe, bg_color, scaling_modifier, pc._xyz.device, size)
    binding = getattr(pc, "binding", None)
    if binding is None:
        return rs, None, (None, None, None)
    if getattr(pc, "face_center", None) is None:
        pc.select_mesh_by_timestep(0)  # as the reference getters do (scene/gaussian_model.py:119-120)
    return rs, binding, (pc.face_center, pc.face_orien_mat, pc.face_scaling)


def render_bound(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, override_color=None, depth_alpha=False):
    """Fused route (see module docstring).  depth_alpha=True adds the differentiable "alpha" and "depth" planes."""
    return _train_frame(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, depth_alpha)


def _train_frame(camera, pc, pipe, bg_color, scaling_modifier, override_color, depth_alpha, size=None):
    """The differentiable fused-route frame of a camera object, or of the views of a (K, 37) device camera table of
    image `size` (W, H) (render_views_train): then every output has a leading K."""
    rs, binding, (fc, fR, fs) = _fused_frame(camera, pc, pipe, bg_color, scaling_modifier, size)
    lead = () if size is None else (int(camera.shape[0]),)
    screenspace_points = torch.zeros(lead + (pc._xyz.shape[0], 3), dtype=pc._xyz.dtype, device=pc._xyz.device,
                                     requires_grad=True)
    raw = (pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc, pc._features_rest, binding, fc, fR, fs)
    if size is None:
        out = rasterize_bound(rs, *raw, means2D=screenspace_points, colors_precomp=override_color, grad_sink=pc,
                              tanfov=getattr(camera, "tanfov", None), depth_alpha=depth_alpha)
    else:
        out = rasterize_bound_views_train(rs, camera, *raw, means2D=screenspace_points, grad_sink=pc,
                                          depth_alpha=depth_alpha)
    rendered_image, radii = out[0], out[1]
    res = {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": _visible(radii),
           "radii": radii}
    if depth_alpha:
        res["alpha"], res["depth"] = out[2], out[3]
    return res


def _forward_only(camera, pc, pipe, bg_color, scaling_modifier, display: bool, float_image: bool,
                  depth_alpha: bool = False, size=None, quantize: str = "render"):
    """Fused route, forward only (no autograd): the float image and/or the display image [and the alpha / depth
    planes] of a camera object, or of the views of a (K, 37) device camera table of image `size` (W, H)
    (render_views, GraphedRender): then every output has a leading K.  quantize: the display image's bytes,
    "render" or "viewer" (rasterizer.rasterize_bound)."""
    if not _has_raw(pc):
        raise ValueError("render_display needs the fused route: a model exposing the raw parameters "
                         "(_xyz, _rotation, _scaling, _opacity, _features_dc, _features_rest)")
    device = pc._xyz.device
    d = lambda t: None if t is None else t.detach()  # noqa: E731  (no gradient: the forward keeps no backward state)
    with torch.no_grad():
        rs, binding, (fc, fR, fs) = _fused_frame(camera, pc, pipe, bg_color, scaling_modifier, size)
        raw = (d(pc._xyz), d(pc._rotation), d(pc._scaling), d(pc._opacity), d(pc._features_dc), d(pc._features_rest),
               binding, d(fc), d(fR), d(fs))
        if size is None:
            rgb8 = torch.empty((rs.image_height, rs.image_width, 3), dtype=torch.uint8, device=device) \
                if display else None
            img, radii, *planes = rasterize_bound(rs, *raw, grad_sink=pc, tanfov=getattr(camera, "tanfov", None),
                                                  rgb8=rgb8, float_image=float_image, depth_alpha=depth_alpha,
                                                  quantize=quantize)
            visible = _visible(radii)
        else:
            img, rgb8, radii, visible, *planes = rasterize_bound_views(
                rs, camera, *raw, hints=view_hints_of(pc), display=display, float_image=float_image,
                depth_alpha=depth_alpha, quantize=quantize)
    res = {"display_u8": rgb8, "render": img, "radii": radii, "visibility_filter": visible}
    if depth_alpha:
        res["alpha"], res["depth"] = planes
    return res


def render_display(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, float_image=False, depth_alpha=False,
                   quantize="render"):
    """One playback frame: the fused route's forward only, no autograd, with the image as the reference's render.py
    and viewers consume it -- `display_u8`, a (H,W,3) uint8 tensor equal bit for bit to
    render(...)["render"].mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8), written by the forward
    blend itself (3 bytes per pixel instead of 12, no eager quantisation chain).  float_image=True also returns the
    float (3,H,W) image as "render" (else None).  Returns {"display_u8", "render", "radii", "visibility_filter"};
    depth_alpha=True adds "alpha" and "depth" (1,H,W) float32, from the same blend (the viewers' opacity / depth modes;
    a normalised depth is depth / alpha).
    quantize="viewer": `display_u8` holds the bytes the reference's local viewer exports instead,
    (np.clip(render, 0, 1) * 255).astype(np.uint8) -- a float32 multiply and truncation, no +0.5 -- from the same blend
    epilogue (not combinable with depth_alpha)."""
    return _forward_only(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, True, float_image, depth_alpha,
                         quantize=quantize)


def camera_table(cameras, device) -> torch.Tensor:
    """(K, 37) float32 device table of camera objects: row k = graph.camera_block(cam_k, fov=True), with the camera's
    device field of view (`cam.tanfov`) when it carries one."""
    from .graph import camera_block
    rows = []
    for cam in cameras:
        row = camera_block(cam, fov=True).to(device)
        tanfov = getattr(cam, "tanfov", None)
        if tanfov is not None:
            row[35:] = tanfov.to(device)
        rows.append(row)
    return torch.stack(rows).contiguous()


def render_views(cameras, pc, pipe, bg_color, scaling_modifier=1.0, float_image=False, width=None, height=None,
                 depth_alpha=False):
    """Every camera of a rig in ONE forward (gab200_forward_views): the fused route, forward only, no autograd.
    `cameras`: a list of camera objects of one image size (each with its own matrices and field of view), or a
    (K, 37) float32 device table of camera_block(cam, fov=True) rows together with `width` and `height`.  Returns
    {"display_u8": (K,H,W,3) uint8, "render": (K,3,H,W) float32 or None (float_image=False), "radii": (K,P) int32,
    "visibility_filter": (K,P) bool}; view k equals render_display(cameras[k], ...) bit for bit.  depth_alpha=True adds
    "alpha" and "depth", (K,1,H,W) float32, view k's those of render_display(cameras[k], ..., depth_alpha=True)."""
    table, W, H = _views_table(cameras, pc, width, height, "render_views")
    return _forward_only(table, pc, pipe, bg_color, scaling_modifier, True, float_image, depth_alpha, (W, H))


def _views_table(cameras, pc, width, height, what):
    """(table, W, H) of render_views' `cameras` argument: camera objects of one size, or a table with its size."""
    if not _has_raw(pc):
        raise ValueError(f"{what} needs the fused route: a model exposing the raw parameters "
                         "(_xyz, _rotation, _scaling, _opacity, _features_dc, _features_rest)")
    device = pc._xyz.device
    if isinstance(cameras, torch.Tensor):
        if width is None or height is None:
            raise ValueError("a camera table carries no image size: give width= and height=")
        return check_camera_table(cameras, device), int(width), int(height)
    cameras = list(cameras)
    if not cameras:
        raise ValueError(f"{what} needs at least one camera")
    sizes = {(int(c.image_width), int(c.image_height)) for c in cameras}
    if len(sizes) != 1:
        raise ValueError(f"{what} renders cameras of one image size, got {sorted(sizes)}")
    (W, H), = sizes
    return camera_table(cameras, device), W, H


def render_views_train(cameras, pc, pipe, bg_color, scaling_modifier=1.0, width=None, height=None, depth_alpha=False):
    """The training form of render_views: every camera of one timestep (the model's current face frame) in ONE
    differentiable forward (gab200_forward_views_train).  Returns render()'s dict with a leading K:
    {"render": (K,3,H,W), "viewspace_points": (K,P,3) holder whose .grad row k is camera k's dL/dmean2D,
    "visibility_filter": (K,P) bool, "radii": (K,P) int32}; view k's image and radii equal render(cameras[k], ...)
    bit for bit.  A loss summed over the views backpropagates, in one backward, the sum of the K single-view
    gradients into the model's parameters and face frame.  depth_alpha=True adds the differentiable "alpha" and "depth"
    planes, (K,1,H,W), view k's those of render(cameras[k], ..., depth_alpha=True): a mask or depth term of every view
    joins the same loss and the same backward."""
    table, W, H = _views_table(cameras, pc, width, height, "render_views_train")
    return _train_frame(table, pc, pipe, bg_color, scaling_modifier, None, depth_alpha, (W, H))


def _visible(radii):
    """`radii > 0` (gaussian_renderer/__init__.py:100): the forward wrote it next to the radii (one byte per splat)."""
    v = visible_of(radii)
    return v if v is not None else radii > 0


def render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, override_color=None, fused=None,
           depth_alpha=False):
    python_paths = bool(getattr(pipe, "compute_cov3D_python", False)) or bool(getattr(pipe, "convert_SHs_python", False))
    if fused is None:
        fused = _has_raw(pc) and not python_paths
    if fused:
        return render_bound(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, depth_alpha)
    if depth_alpha:
        raise ValueError("depth_alpha=True needs the fused route (render_bound / rasterize_bound on a model exposing the "
                         "raw parameters, without compute_cov3D_python / convert_SHs_python): the reference route's "
                         "GaussianRasterizer returns only (color, radii)")

    # ---- reference route (data flow of gaussian_renderer/__init__.py:27-101) ----
    if getattr(viewpoint_camera, "tanfov", None) is not None:
        raise ValueError("a camera with a device field of view (cam.tanfov) needs the fused route: the reference route "
                         "only takes FoVx / FoVy as host floats")
    xyz = pc.get_xyz
    device = xyz.device
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    rs = _settings(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, device)
    rasterizer = GaussianRasterizer(raster_settings=rs, hints=hints_of(pc))
    means3D, means2D, opacity = xyz, screenspace_points, pc.get_opacity
    scales = rotations = cov3D_precomp = None
    if getattr(pipe, "compute_cov3D_python", False):
        cov3D_precomp = pc.get_covariance(scaling_modifier)
    else:
        scales, rotations = pc.get_scaling, pc.get_rotation
    shs = colors_precomp = None
    if override_color is None:
        if getattr(pipe, "convert_SHs_python", False):
            from .sh import eval_sh
            shs_view = pc.get_features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
            dir_pp = xyz - rs.campos.repeat(pc.get_features.shape[0], 1)
            dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
            sh2rgb = eval_sh(pc.active_sh_degree, shs_view, dir_pp_normalized)
            colors_precomp = torch.clamp_min(sh2rgb + 0.5, 0.0)
        else:
            shs = pc.get_features
    else:
        colors_precomp = override_color
    rendered_image, radii = rasterizer(means3D=means3D, means2D=means2D, shs=shs, colors_precomp=colors_precomp,
                                       opacities=opacity, scales=scales, rotations=rotations,
                                       cov3D_precomp=cov3D_precomp)
    return {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": _visible(radii),
            "radii": radii}
