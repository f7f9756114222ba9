"""gaussianavatars_b200 -- H100-native (sm_90a) differentiable Gaussian-splat rasterizer with the GaussianAvatars
FLAME mesh binding fused into preprocess.  Drop-in for the `diff_gaussian_rasterization` operator behind
gaussian_renderer.render() (reference: gaussian_renderer/__init__.py:15,37-52,86-94).

Nothing here falls back to CPU or eager PyTorch: the ops raise if libgaussianavatars_b200.so is missing.
"""
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians, rasterize_bound,
                         bind_activate, set_exact_binning, face_frame, l1_loss_u8)
from .renderer import render, render_bound, render_display, render_views, render_views_train
from .training import photometric_loss, image_metrics, Adam, binding_regularizers, expon_lr_schedule, composite_rgba
from .frames import FrameStore
from .schedule import ViewSchedule, epoch_order
from .io import load_ply, save_ply, load_flame_param, save_flame_param
from .densify import densify_and_prune, densify_arrays, add_densification_stats
from .flame import FlameLBS, flame_pose, flame_param_groups
from .mesh import mesh_overlay, MeshRenderer
from .lpips import LpipsNet, lpips, launch_lpips, lpips_features

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "rasterize_bound",
           "bind_activate", "set_exact_binning", "face_frame", "l1_loss_u8", "render", "render_bound", "render_display", "render_views",
           "render_views_train",
           "photometric_loss", "image_metrics", "Adam", "binding_regularizers", "load_ply", "save_ply", "load_flame_param", "save_flame_param", "densify_and_prune", "densify_arrays",
           "add_densification_stats", "expon_lr_schedule", "FlameLBS", "flame_pose", "flame_param_groups",
           "mesh_overlay", "MeshRenderer", "composite_rgba", "FrameStore",
           "ViewSchedule", "epoch_order", "LpipsNet", "lpips", "launch_lpips", "lpips_features"]
