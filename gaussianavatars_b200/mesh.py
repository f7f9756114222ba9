"""The tracked mesh drawn over an image on the device (csrc/mesh.cu): what the reference's mesh renderer
(mesh_renderer/__init__.py) asks of nvdiffrast, and render.py's mesh composite (render.py:75-81), fused.

    frame = mesh_overlay(pc.verts, pc.faces, view, gt_u8)       # render.py --render_mesh: (H,W,3) uint8 bytes
    frames = mesh_overlay_views(pc.verts, pc.faces, cams, gts)  # K cameras of one timestep: (K,H,W,3), one call

`mesh_overlay` renders at the camera's (H,W), as the reference's `use_opengl=True` path does.  Its default CUDA context
renders at (H//8*8, W//8*8) -- or 2048x2048 when a side exceeds 2048 -- and resizes bilinearly; the two agree whenever W
and H are multiples of 8 and at most 2048 (720p, 1080p).  The nvdiffrast shim (compat/nvdiffrast) runs the reference's
own code, resize included.  Nothing here is differentiable: inputs that require grad are detached.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _native as N

LIGHTING = {"front": N.MESH_LIGHT_FRONT, "constant": N.MESH_LIGHT_CONSTANT}


def mesh_adjacency(faces: torch.Tensor) -> torch.Tensor:
    """(F,3) int32 on faces' device: adjacency[f, k] = the face across edge k = (faces[f,k], faces[f,(k+1)%3]), or -1 when
    no other face -- or more than one -- shares that edge.  A sort of the packed (min, max) vertex keys of the 3F
    edges; an edge key shared by exactly two entries pairs them."""
    f = faces.detach().long()
    F = f.shape[0]
    a = f
    b = f[:, [1, 2, 0]]
    lo, hi = torch.minimum(a, b).reshape(-1), torch.maximum(a, b).reshape(-1)
    key = lo * (1 << 31) + hi  # vertex indices are int32: the packed key fits in int64, no host read of max()
    ks, order = torch.sort(key, stable=True)
    _, inv, counts = torch.unique_consecutive(ks, return_inverse=True, return_counts=True)
    pair = counts[inv] == 2
    first = torch.zeros_like(pair)
    first[:-1] = pair[:-1] & (ks[1:] == ks[:-1])
    adj_sorted = torch.full_like(order, -1)
    i = torch.nonzero(first).squeeze(1)
    adj_sorted[i] = order[i + 1] // 3
    adj_sorted[i + 1] = order[i] // 3
    adj = torch.empty_like(adj_sorted)
    adj[order] = adj_sorted
    return adj.reshape(F, 3).to(torch.int32)


class _AdjacencyCache:
    """One faces tensor's adjacency, rebuilt when the tensor (identity) or its contents (_version) change."""

    def __init__(self):
        self.key = None
        self.adj = None

    def get(self, faces: torch.Tensor) -> torch.Tensor:
        key = (faces, faces._version)
        if self.key is None or self.key[0] is not faces or self.key[1] != faces._version:
            self.adj = mesh_adjacency(faces)
            self.key = key
        return self.adj


_overlay_adjacency = _AdjacencyCache()


def _faces_i32(faces: torch.Tensor, device) -> torch.Tensor:
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.shape[0] < 1:
        raise ValueError(f"faces must be (F,3) with F >= 1, got {tuple(faces.shape)}")
    if faces.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"faces must be int32 or int64, got {faces.dtype}")
    return faces.detach().to(device=device, dtype=torch.int32).contiguous()


def _check_size(W: int, H: int):
    if not (1 <= W <= N.MESH_MAX_SIDE and 1 <= H <= N.MESH_MAX_SIDE):
        raise ValueError(f"image size {W}x{H} outside [1, {N.MESH_MAX_SIDE}]")


def _camera_floats(camera, device) -> torch.Tensor:
    if isinstance(camera, torch.Tensor):
        blk = camera.detach().reshape(-1)
        if blk.numel() not in (35, 37) or blk.dtype != torch.float32:
            raise ValueError("a camera block is 35 or 37 float32 values (graph.camera_block)")
        return blk.to(device).contiguous()
    from .graph import camera_block

    return camera_block(camera).to(device).contiguous()


def launch_mesh(*, verts, faces, width, height, pos_kind=N.MESH_POS_WORLD, camera=None, adjacency=None,
                face_colors=None, background=(1.0, 1.0, 1.0), lighting="front", antialias=True, base=None,
                opacity=None, out_u8=None, out_float=None, out_rgba=None, out_rast=None, in_rast=None, in_color=None,
                out_color=None, error_flag=None, stream=None, views=None, quantize="render"):
    """One gab200_mesh_render call on device tensors (no checks beyond the library's own); returns nothing.
    views=K: one gab200_mesh_render_views call instead -- camera a (K,37) table, base (K,3,H,W), out_u8 (K,H,W,3).
    quantize: how out_u8 is quantised, "render" (render.py's bytes) or "viewer" (the local viewer's export)."""
    dev = verts.device
    F = faces.shape[0]
    _check_size(width, height)
    if lighting not in LIGHTING:
        raise ValueError(f"lighting must be one of {sorted(LIGHTING)}, got {lighting!r}")
    a = N.MeshArgs()
    a.abi_version, a.V, a.F, a.width, a.height = N.ABI_VERSION, verts.shape[0], F, width, height
    a.pos_kind = pos_kind
    a.verts, a.faces, a.adjacency, a.camera = N.ptr(verts), N.ptr(faces), N.ptr(adjacency), N.ptr(camera)
    a.face_colors = N.ptr(face_colors)
    a.background = (C.c_float * 3)(*[float(x) for x in background])
    a.lighting, a.antialias = LIGHTING[lighting], int(bool(antialias))
    if base is None:
        a.base_kind = N.MESH_BASE_NONE
    else:
        a.base_kind = N.MESH_BASE_U8_CHW if base.dtype == torch.uint8 else N.MESH_BASE_FLOAT_CHW
    a.base, a.opacity = N.ptr(base), N.ptr(opacity)
    a.out_u8, a.out_float, a.out_rgba, a.out_rast = N.ptr(out_u8), N.ptr(out_float), N.ptr(out_rgba), N.ptr(out_rast)
    a.in_rast, a.in_color, a.out_color = N.ptr(in_rast), N.ptr(in_color), N.ptr(out_color)
    a.channels = 0 if in_color is None else in_color.shape[-1]
    a.quantize = N.quantize_mode(quantize)
    a.error_flag = N.ptr(error_flag)
    L = N.lib()
    nbytes = L.gab200_mesh_scratch_bytes(F, width, height) if views is None else \
        L.gab200_mesh_views_scratch_bytes(int(views), F, width, height)
    scratch = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)
    a.scratch = scratch.data_ptr()
    s = torch.cuda.current_stream(dev) if stream is None else stream
    if views is None:
        N.check(L.gab200_mesh_render(C.byref(a), C.c_void_p(s.cuda_stream)), "gab200_mesh_render")
    else:
        N.check(L.gab200_mesh_render_views(C.byref(a), int(views), C.c_void_p(s.cuda_stream)),
                "gab200_mesh_render_views")


def opacity_pair(mesh_opacity: float, device) -> torch.Tensor:
    """{o, 1 - o} as float32, both rounded from Python doubles: the scalars torch forms for render.py's expression."""
    o = float(mesh_opacity)
    return torch.tensor([o, 1.0 - o], dtype=torch.float32, device=device)


def _verts_v3(verts: torch.Tensor) -> torch.Tensor:
    v = verts.detach()
    if v.dim() == 3:
        if v.shape[0] != 1:
            raise ValueError(f"one mesh per call: verts batch {v.shape[0]}")
        v = v[0]
    if v.dim() != 2 or v.shape[1] != 3 or v.shape[0] < 1:
        raise ValueError(f"verts must be (V,3) or (1,V,3), got {tuple(verts.shape)}")
    if v.dtype != torch.float32:
        raise TypeError(f"verts must be float32, got {v.dtype}")
    if not v.is_cuda:
        raise RuntimeError("gaussianavatars_b200 has no CPU path: verts must be on a CUDA device")
    return v.contiguous()


def _face_colors(face_colors, F, device):
    if face_colors is None:
        return None
    fc = face_colors.detach()
    if fc.dim() == 3:
        if fc.shape[0] != 1:
            raise ValueError(f"one mesh per call: face_colors batch {fc.shape[0]}")
        fc = fc[0]
    if tuple(fc.shape) != (F, 3):
        raise ValueError(f"face_colors must be ({F},3) or (1,{F},3), got {tuple(face_colors.shape)}")
    return fc.to(device=device, dtype=torch.float32).contiguous()


def mesh_overlay(verts: torch.Tensor, faces: torch.Tensor, camera, base: torch.Tensor, mesh_opacity: float = 0.5,
                 face_colors: Optional[torch.Tensor] = None, background: Sequence[float] = (1.0, 1.0, 1.0),
                 lighting: str = "front", antialias: bool = True, out: str = "u8",
                 error_flag: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The mesh at `mesh_opacity` over `base`, as render.py composes its renders_mesh frames:
        rgb_mesh * a * o + base * (a * (1 - o) + (1 - a))
    verts (V,3) | (1,V,3) float32; faces (F,3) int; camera: a camera object or a 35/37-float camera block
    (graph.camera_block); base (3,H,W) float32, or uint8 read as value/255 (the ground-truth bytes).
    out="u8": (H,W,3) uint8 quantised as render.py does before it writes a PNG; out="float": (3,H,W) float32.
    error_flag: optional device int32 into which 1 is ORed when a face index is outside [0, V) (that face is skipped)."""
    if out not in ("u8", "float"):
        raise ValueError(f"out must be 'u8' or 'float', got {out!r}")
    v = _verts_v3(verts)
    dev = v.device
    if base.dim() != 3 or base.shape[0] != 3 or base.dtype not in (torch.float32, torch.uint8):
        raise ValueError(f"base must be (3,H,W) float32 or uint8, got {tuple(base.shape)} {base.dtype}")
    H, W = int(base.shape[1]), int(base.shape[2])
    if not isinstance(camera, torch.Tensor) and (int(camera.image_width), int(camera.image_height)) != (W, H):
        raise ValueError(f"camera is {camera.image_width}x{camera.image_height}, base is {W}x{H}")
    f = _faces_i32(faces, dev)
    adj = _overlay_adjacency.get(faces).to(dev) if antialias else None
    result = (torch.empty(H, W, 3, dtype=torch.uint8, device=dev) if out == "u8"
              else torch.empty(3, H, W, dtype=torch.float32, device=dev))
    launch_mesh(verts=v, faces=f, width=W, height=H, camera=_camera_floats(camera, dev), adjacency=adj,
                face_colors=_face_colors(face_colors, f.shape[0], dev), background=background, lighting=lighting,
                antialias=antialias, base=base.detach().to(dev).contiguous(), opacity=opacity_pair(mesh_opacity, dev),
                out_u8=result if out == "u8" else None, out_float=result if out == "float" else None,
                error_flag=error_flag)
    return result


def _check_cameras(cameras, K: int, W: int, H: int):
    """K camera objects of the base's size, or a (K,37) float32 table; returns the objects' list, or the table."""
    if isinstance(cameras, torch.Tensor):
        if tuple(cameras.shape) != (K, N.CAMERA_FLOATS) or cameras.dtype != torch.float32:
            raise ValueError(f"the camera table of {K} views is ({K},{N.CAMERA_FLOATS}) float32 "
                             f"(renderer.camera_table), got {tuple(cameras.shape)} {cameras.dtype}")
        return cameras.detach()
    cams = list(cameras)
    if len(cams) != K:
        raise ValueError(f"{len(cams)} cameras for {K} base planes")
    for c in cams:
        if (int(c.image_width), int(c.image_height)) != (W, H):
            raise ValueError(f"a camera is {c.image_width}x{c.image_height}, base is {W}x{H}")
    return cams


def mesh_overlay_views(verts: torch.Tensor, faces: torch.Tensor, cameras, base: torch.Tensor,
                       mesh_opacity: float = 0.5, face_colors: Optional[torch.Tensor] = None,
                       background: Sequence[float] = (1.0, 1.0, 1.0), lighting: str = "front", antialias: bool = True,
                       error_flag: Optional[torch.Tensor] = None) -> torch.Tensor:
    """mesh_overlay under K cameras of one vertex set in one call (gab200_mesh_render_views): frame k is bit for bit
    mesh_overlay(verts, faces, cameras[k], base[k], ...) with out="u8".
    cameras: K camera objects of the base's size, or a (K,37) float32 table (renderer.camera_table); base (K,3,H,W)
    float32, or uint8 read as value/255.  Returns (K,H,W,3) uint8.  The scratch holds K winner maps: K * 8 * H * W
    bytes and more (~265 MB for K = 16 at 1080p)."""
    if base.dim() != 4 or base.shape[1] != 3 or base.dtype not in (torch.float32, torch.uint8):
        raise ValueError(f"base must be (K,3,H,W) float32 or uint8, got {tuple(base.shape)} {base.dtype}")
    K, H, W = int(base.shape[0]), int(base.shape[2]), int(base.shape[3])
    if not 1 <= K <= N.MAX_VIEWS:
        raise ValueError(f"base holds 1 .. {N.MAX_VIEWS} views, got {K}")
    _check_size(W, H)
    cams = _check_cameras(cameras, K, W, H)
    v = _verts_v3(verts)
    dev = v.device
    if isinstance(cams, torch.Tensor):
        table = cams.to(dev).contiguous()
    else:
        from .renderer import camera_table

        table = camera_table(cams, dev)
    f = _faces_i32(faces, dev)
    adj = _overlay_adjacency.get(faces).to(dev) if antialias else None
    result = torch.empty(K, H, W, 3, dtype=torch.uint8, device=dev)
    launch_mesh(verts=v, faces=f, width=W, height=H, camera=table, adjacency=adj,
                face_colors=_face_colors(face_colors, f.shape[0], dev), background=background, lighting=lighting,
                antialias=antialias, base=base.detach().to(dev).contiguous(), opacity=opacity_pair(mesh_opacity, dev),
                out_u8=result, error_flag=error_flag, views=K)
    return result


class MeshRenderer:
    """The reference's NVDiffRenderer.render_from_camera on this library's kernels, rendered at the camera's (H,W)
    (the reference's use_opengl=True path).  Returns its dict {albedo, normal, diffuse, rgba}, each (1,H,W,3|4), row 0
    at the top; rgba is antialiased, the other three are not (as in the reference)."""

    def __init__(self, lighting_type: str = "front"):
        if lighting_type not in LIGHTING:
            raise NotImplementedError(f"Unknown lighting type: {lighting_type}")
        self.lighting_type = lighting_type
        self._adjacency = _AdjacencyCache()

    def render_from_camera(self, verts, faces, cam, background_color=(1.0, 1.0, 1.0), face_colors=None):
        if not isinstance(background_color, (list, tuple)) or len(background_color) != 3:
            raise ValueError("background_color must be three floats")
        v = _verts_v3(verts)
        dev = v.device
        W, H = int(cam.image_width), int(cam.image_height)
        f = _faces_i32(faces, dev)
        F = f.shape[0]
        fc = _face_colors(face_colors, F, dev)
        rgba = torch.empty(H, W, 4, dtype=torch.float32, device=dev)
        rast = torch.empty(H, W, 4, dtype=torch.float32, device=dev)
        launch_mesh(verts=v, faces=f, width=W, height=H, camera=_camera_floats(cam, dev),
                    adjacency=self._adjacency.get(faces).to(dev), face_colors=fc, background=background_color,
                    lighting=self.lighting_type, antialias=True, out_rgba=rgba, out_rast=rast)
        # the un-antialiased maps of the reference's dict: per-face quantities gathered by the winner index
        fg = rast[..., 3:] > 0
        fid = (rast[..., 3].long() - 1).clamp_min(0)
        wv = cam.world_view_transform.detach().to(dev, torch.float32).clone()
        wv[:, 1] = -wv[:, 1]
        wv[:, 2] = -wv[:, 2]
        vc = torch.cat([v, torch.ones_like(v[:, :1])], 1) @ wv
        fl = f.long()
        v0, v1, v2 = vc[fl[:, 0], :3], vc[fl[:, 1], :3], vc[fl[:, 2], :3]
        n = torch.cross(v1 - v0, v2 - v0, dim=-1)
        n = n / torch.sqrt(torch.clamp((n * n).sum(-1, keepdim=True), min=1e-20))
        normal = n[fid]
        diffuse = (torch.ones_like(normal) if self.lighting_type == "constant"
                   else torch.clamp(normal[..., 2:3], 0.0, 1.0))
        albedo = fc[fid] if fc is not None else torch.ones_like(normal)
        bg = torch.tensor(list(background_color), dtype=torch.float32, device=dev)
        return {"albedo": albedo[None], "normal": torch.where(fg, normal, bg)[None],
                "diffuse": torch.where(fg, diffuse, bg)[None], "rgba": rgba[None]}
