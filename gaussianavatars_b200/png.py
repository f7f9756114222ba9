"""PNG files written on the device: what render.py's `Image.fromarray(data).save(path)` does per view, as six kernels.

    data = encode_png(display)                 # (H,W,3) uint8 CUDA tensor -> the bytes of a PNG file
    files = encode_png(displays)               # (K,H,W,3) -> K files
    open(path, "wb").write(data)

    player = GraphedRender(pc, W, H, bg, png=True, host_slots=2)   # the encode inside the captured replay
    player.run(); open(path, "wb").write(player.host_png())

Each file is an 8-bit RGB PNG (signature, IHDR, one IDAT, IEND) that PIL and zlib open; its pixels are the input bytes.
Each row gets the PNG filter with the least sum of |signed byte| (libpng's heuristic; oracle/png.py restates it), and
the filtered stream is deflated in 32 KiB segments, each the smallest of a dynamic, fixed or stored block
(include/gab200_rasterizer.h, gab200_png_encode).  The bytes differ from PIL's; the same input always gives the
same file.  No file exceeds png_bound(W, H), so the output capacity is fixed per (K, W, H) and the encode is
capturable.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _native as N


def png_bound(width: int, height: int) -> int:
    """The largest file a width x height image can take (gab200_png_bound)."""
    b = int(N.lib().gab200_png_bound(int(width), int(height)))
    if b < 0:
        raise ValueError(f"no PNG of {width}x{height}: the size must be positive and its IDAT fit 2^31 - 1 bytes")
    return b


def slot_stride(width: int, height: int) -> int:
    """Bytes per file in an output buffer: the bound rounded up to 16 (gab200_png_copy moves 16-byte words)."""
    return (png_bound(width, height) + 15) // 16 * 16


def check_u8(u8, name: str = "u8") -> tuple:
    """(K, H, W) of a CUDA uint8 (H,W,3) or (K,H,W,3) contiguous tensor; raises naming what is wrong."""
    if not isinstance(u8, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(u8).__name__}")
    if u8.dtype != torch.uint8:
        raise ValueError(f"{name} must be uint8 (display bytes), got {u8.dtype}")
    if u8.dim() not in (3, 4) or u8.shape[-1] != 3:
        raise ValueError(f"{name} must be (H, W, 3) or (K, H, W, 3), got shape {tuple(u8.shape)}")
    if not u8.is_contiguous():
        raise ValueError(f"{name} must be contiguous (rows of 3W bytes); call .contiguous() first")
    if u8.device.type != "cuda":
        raise ValueError(f"{name} must be on a CUDA device (the encode runs there), got {u8.device}")
    K = 1 if u8.dim() == 3 else int(u8.shape[0])
    H, W = int(u8.shape[-3]), int(u8.shape[-2])
    if K < 1 or H < 1 or W < 1:
        raise ValueError(f"{name} must hold at least one pixel per image, got shape {tuple(u8.shape)}")
    png_bound(W, H)
    return K, H, W


def scratch(K: int, H: int, W: int, device) -> torch.Tensor:
    """The scratch of an encode of K images of H x W (gab200_png_scratch_bytes), 256-byte aligned."""
    n = int(N.lib().gab200_png_scratch_bytes(K, H, W))
    if n == 0:
        raise ValueError(f"no PNG encode of {K} views of {W}x{H}")
    return torch.empty(n, dtype=torch.uint8, device=device)   # the caching allocator aligns to 512 bytes


def launch_encode(u8: torch.Tensor, scratch_buf: torch.Tensor, out: torch.Tensor, out_len: torch.Tensor):
    """Enqueues gab200_png_encode on the current stream: u8 (K,H,W,3) or (H,W,3) -> file k in out[k] ((K, stride)
    uint8), its length in out_len[k] ((K,) int64).  Reads nothing on the host: capturable."""
    K, H, W = check_u8(u8)
    if out.dtype != torch.uint8 or out.dim() != 2 or out.shape[0] != K or out.shape[1] < png_bound(W, H) or \
            not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 ({K}, >= {png_bound(W, H)}) tensor")
    if out_len.dtype != torch.int64 or tuple(out_len.shape) != (K,):
        raise ValueError(f"out_len must be an int64 ({K},) tensor")
    stream = C.c_void_p(torch.cuda.current_stream(u8.device).cuda_stream)
    N.check(N.lib().gab200_png_encode(K, H, W, u8.data_ptr(), scratch_buf.data_ptr(), out.data_ptr(), out.stride(0),
                                      out_len.data_ptr(), stream), "gab200_png_encode")


def launch_copy(src: torch.Tensor, src_len: torch.Tensor, dst: torch.Tensor, dst_len: torch.Tensor, flag=None):
    """Enqueues gab200_png_copy on the current stream: the files of src ((K, stride) uint8) and their lengths ->
    dst / dst_len (device tensors or pinned host tensors, written through their mapped addresses); with `flag` (a
    device int32, the sticky overflow flag of a capture slot) set, no bytes and length -1."""
    K = int(src.shape[0])
    stream = C.c_void_p(torch.cuda.current_stream(src.device).cuda_stream)
    N.check(N.lib().gab200_png_copy(K, src.data_ptr(), src.stride(0), src_len.data_ptr(), N.ptr(flag), dst.data_ptr(),
                                    dst.stride(0), dst_len.data_ptr(), stream), "gab200_png_copy")


@torch.no_grad()
def encode_png(u8: torch.Tensor):
    """The PNG file of a CUDA uint8 (H,W,3) image as `bytes`, or a list of K files of a (K,H,W,3) batch -- render.py's
    display frames, its ground-truth images, or mesh_overlay() output.  Synchronises once to learn the lengths."""
    K, H, W = check_u8(u8)
    dev = u8.device
    with torch.cuda.device(dev):
        out = torch.empty((K, slot_stride(W, H)), dtype=torch.uint8, device=dev)
        out_len = torch.empty(K, dtype=torch.int64, device=dev)
        launch_encode(u8, scratch(K, H, W, dev), out, out_len)
        lens = out_len.tolist()
        files = [out[k, :lens[k]].cpu().numpy().tobytes() for k in range(K)]
    return files[0] if u8.dim() == 3 else files
