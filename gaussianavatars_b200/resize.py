"""The reference loader's resize on the device: Pillow's bicubic `Image.resize`, bit for bit, and the size rule that
picks its target.

    w, h = loader_size(3208, 2200)               # utils/camera_utils.py loadCam, --resolution -1: (1600, 1097)
    out = resize_u8(planes, w, h)                # CUDA uint8 (..., H, W) -> (..., h, w): PIL's bytes

    store = FrameStore(w, h, bg)
    store.add_png(paths, resize=True)            # decode, composite at the file's size, resize: the loader's frames

The reference's CameraDataset.__getitem__ composites each RGBA frame onto the background at the file's size, then
PILtoTorch resizes the "RGB" result to the camera's size with PIL's default filter, BICUBIC (a = -0.5, 22-bit
fixed-point weights; include/gab200_rasterizer.h gab200_resize_u8 and oracle/resize.py state the arithmetic).  Each
plane here is resized as PIL resizes an "L" image, which is also what it does to each channel of an "RGB" image.
Pillow 7 and later; earlier versions resized with NEAREST by default.
"""
from __future__ import annotations

import ctypes as C
import numbers

import torch

from . import _native as N

LOADER_MAX_WIDTH = 1600   # loadCam's --resolution -1 rescales wider captures to this width


def loader_size(width: int, height: int, resolution=-1, resolution_scale: float = 1.0) -> tuple:
    """(width, height) the reference trains a width x height capture at: loadCam's rule (utils/camera_utils.py:20-40).

    resolution 1, 2, 4 or 8 divides both sides by resolution * resolution_scale and rounds (Python's round: halves to
    even).  -1 (the default) rescales a capture wider than 1600 pixels to width 1600 and keeps any other; another value
    is the target width.  Those two scale both sides by one float factor and truncate, so 1601 x 1200 -> 1599 x 1199."""
    orig_w, orig_h = int(width), int(height)
    if orig_w < 1 or orig_h < 1:
        raise ValueError(f"a capture has a positive size, got {orig_w}x{orig_h}")
    if isinstance(resolution, bool) or not isinstance(resolution, numbers.Real):
        raise TypeError(f"resolution must be a number, got {type(resolution).__name__}")
    if resolution in [1, 2, 4, 8]:
        w = round(orig_w / (resolution_scale * resolution))
        h = round(orig_h / (resolution_scale * resolution))
    else:
        if resolution == -1:
            global_down = orig_w / LOADER_MAX_WIDTH if orig_w > LOADER_MAX_WIDTH else 1
        elif resolution > 0:
            global_down = orig_w / resolution
        else:
            raise ValueError(f"resolution must be -1, 1, 2, 4, 8 or a positive target width, got {resolution!r}")
        scale = float(global_down) * float(resolution_scale)
        w, h = int(orig_w / scale), int(orig_h / scale)
    if w < 1 or h < 1:
        raise ValueError(f"{orig_w}x{orig_h} at resolution {resolution!r}, scale {resolution_scale!r} is {w}x{h}: "
                         "no pixel left")
    return w, h


def check_size(size) -> tuple:
    """(width, height) of a target size given as two positive ints."""
    try:
        w, h = size
    except (TypeError, ValueError):
        raise TypeError(f"size must be (width, height), got {size!r}") from None
    for v in (w, h):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < 1:
            raise ValueError(f"size must be two positive ints (width, height), got {size!r}")
    return int(w), int(h)


def _check_planes(t, name: str):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() < 2:
        raise TypeError(f"{name} must be a uint8 (..., H, W) tensor, got {getattr(t, 'dtype', type(t))} "
                        f"{tuple(getattr(t, 'shape', ()))}")
    if t.device.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: tensors must be CUDA tensors")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def scratch_bytes(planes: int, in_h: int, in_w: int, out_h: int, out_w: int) -> int:
    """Bytes of a resize's scratch (gab200_resize_scratch_bytes); raises for sizes the resize refuses."""
    n = int(N.lib().gab200_resize_scratch_bytes(planes, in_h, in_w, out_h, out_w))
    if n == 0:
        raise ValueError(f"no resize of {planes} planes of {in_w}x{in_h} to {out_w}x{out_h}")
    return n


def launch_resize(src: torch.Tensor, dst: torch.Tensor, scratch: torch.Tensor):
    """Enqueues gab200_resize_u8 on the current stream: src (..., H, W) -> dst (..., h, w), both contiguous uint8 on
    one device with the same leading shape; scratch: scratch_bytes(...) uint8 on that device.  Reads nothing on the
    host and allocates nothing: capturable."""
    _check_planes(src, "src")
    _check_planes(dst, "dst")
    if dst.shape[:-2] != src.shape[:-2] or dst.device != src.device:
        raise ValueError(f"dst must be (..., h, w) with src's leading shape {tuple(src.shape[:-2])} on {src.device}, "
                         f"got {tuple(dst.shape)} on {dst.device}")
    H, W, h, w = int(src.shape[-2]), int(src.shape[-1]), int(dst.shape[-2]), int(dst.shape[-1])
    planes = src.numel() // max(H * W, 1)
    need = scratch_bytes(planes, H, W, h, w)
    if scratch.dtype != torch.uint8 or scratch.numel() < need or scratch.device != src.device:
        raise ValueError(f"scratch must hold {need} uint8 bytes on {src.device}")
    with torch.cuda.device(src.device):
        stream = torch.cuda.current_stream(src.device).cuda_stream
        N.check(N.lib().gab200_resize_u8(planes, H, W, h, w, src.data_ptr(), dst.data_ptr(), scratch.data_ptr(),
                                         C.c_void_p(stream)), "gab200_resize_u8")
    return dst


@torch.no_grad()
def resize_u8(planes: torch.Tensor, width: int, height: int) -> torch.Tensor:
    """A CUDA uint8 (..., H, W) tensor of planes resized to (..., height, width) on the device: each plane the bytes
    of PIL's `Image.fromarray(plane, "L").resize((width, height))` -- and so each channel of an "RGB" image's resize.
    A strided input is made contiguous first.  Capturable (its outputs come from the current graph's pool)."""
    if isinstance(planes, torch.Tensor) and planes.device.type == "cuda":
        planes = planes.contiguous()
    _check_planes(planes, "planes")
    width, height = check_size((width, height))
    H, W = int(planes.shape[-2]), int(planes.shape[-1])
    if H < 1 or W < 1:
        raise ValueError(f"planes must hold at least one pixel each, got shape {tuple(planes.shape)}")
    n = planes.numel() // (H * W)
    dev = planes.device
    out = torch.empty(planes.shape[:-2] + (height, width), dtype=torch.uint8, device=dev)
    if n == 0:
        return out
    scratch = torch.empty(scratch_bytes(n, H, W, height, width), dtype=torch.uint8, device=dev)
    return launch_resize(planes, out, scratch)
