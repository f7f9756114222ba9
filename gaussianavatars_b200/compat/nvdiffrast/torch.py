"""nvdiffrast.torch's rasterize / antialias on this library's mesh kernels (csrc/mesh.cu), in nvdiffrast's documented
layouts, so the reference's mesh_renderer -- and through it render.py --render_mesh and the viewers' mesh overlay --
runs unmodified:
  rasterize(glctx, pos, tri, resolution) -> (rast_out, rast_db): rast_out [1,H,W,4] = perspective-correct barycentrics
    (u, v) of the triangle's vertices 0 and 1, z/w, triangle index + 1 (0 where nothing is covered), row 0 at clip
    y = -1; rast_db is zeros.
  antialias(color, rast, pos, tri) -> [1,H,W,C]: the silhouette antialiasing of include/gab200_rasterizer.h.
Only one image per call (B = 1, all the reference uses), no `ranges`, no gradients (no caller differentiates through
the mesh render): inputs that require grad are detached."""
import os
import sys

_root = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", "..", ".."))
if _root not in sys.path:
    sys.path.insert(0, _root)

import torch  # noqa: E402

from gaussianavatars_b200 import _native as _N  # noqa: E402
from gaussianavatars_b200.mesh import launch_mesh, mesh_adjacency  # noqa: E402


class RasterizeCudaContext:
    def __init__(self, device=None):
        self.device = device


class RasterizeGLContext:
    def __init__(self, output_db=True, mode="automatic", device=None):
        self.output_db = output_db
        self.device = device


def _pos_tri(pos, tri):
    if pos.dim() != 3 or pos.shape[0] != 1 or pos.shape[2] != 4:
        raise ValueError(f"pos must be [1, V, 4] (one image per call), got {tuple(pos.shape)}")
    if pos.dtype != torch.float32 or not pos.is_cuda:
        raise TypeError("pos must be a float32 CUDA tensor")
    if tri.dim() != 2 or tri.shape[1] != 3 or tri.shape[0] < 1 or tri.dtype != torch.int32:
        raise ValueError(f"tri must be [F, 3] int32 with F >= 1, got {tuple(tri.shape)} {tri.dtype}")
    return pos.detach()[0].contiguous(), tri.detach().to(pos.device).contiguous()


def rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    if ranges is not None:
        raise NotImplementedError("rasterize: range mode (ranges=) is not supported")
    p, t = _pos_tri(pos, tri)
    h, w = int(resolution[0]), int(resolution[1])
    rast = torch.empty(1, h, w, 4, dtype=torch.float32, device=p.device)
    launch_mesh(verts=p, faces=t, width=w, height=h, pos_kind=_N.MESH_POS_CLIP, antialias=False, out_rast=rast)
    return rast, torch.zeros_like(rast)


def antialias(color, rast, pos, tri, topology_hash=None, pos_gradient_boost=1.0):
    p, t = _pos_tri(pos, tri)
    if color.dim() != 4 or color.shape[0] != 1 or color.dtype != torch.float32:
        raise ValueError(f"color must be float32 [1, H, W, C], got {tuple(color.shape)} {color.dtype}")
    _, h, w, c = color.shape
    if tuple(rast.shape) != (1, h, w, 4):
        raise ValueError(f"rast must be [1, {h}, {w}, 4], got {tuple(rast.shape)}")
    out = torch.empty_like(color, memory_format=torch.contiguous_format)
    launch_mesh(verts=p, faces=t, width=w, height=h, pos_kind=_N.MESH_POS_CLIP, adjacency=mesh_adjacency(t),
                antialias=True, in_rast=rast.detach().contiguous(), in_color=color.detach().contiguous(),
                out_color=out)
    return out
