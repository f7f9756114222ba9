"""PNG files written and read on the device: what render.py's `Image.fromarray(data).save(path)` does per view, as six
kernels, and what the loader's and metrics.py's `Image.open(path)` do, as two.

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

    rgba = decode_png(paths)                   # F files of one size -> (F,H,W,4) uint8 CUDA tensor
    rgb = decode_png(data, channels=3)         # one file (bytes or a path) -> (H,W,3)

decode_png reads 8-bit RGB and RGBA files, not interlaced (include/gab200_rasterizer.h, gab200_png_decode): the host
walks the chunks and checks IHDR and the CRC of every chunk before the image data, the IDAT data of all files goes to
the device in one copy, and one launch inflates and unfilters them.  The pixels equal PIL's `convert("RGBA")` (or its
first three channels).  Stricter than PIL: a file whose data is truncated or inflates past the image is refused.
"""
from __future__ import annotations

import ctypes as C
import os
import struct
import zlib

import numpy as np
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


# ---- decode ------------------------------------------------------------------------------------------------------
SIGNATURE = b"\x89PNG\r\n\x1a\n"
COLOR_TYPES = {0: "grey", 2: "RGB", 3: "palette", 4: "grey+alpha", 6: "RGBA"}


def _read(f, i: int) -> tuple:
    """(bytes, name) of file i: a path is read, a bytes-like object is taken as the file's bytes."""
    if isinstance(f, (str, os.PathLike)):
        with open(f, "rb") as fh:
            return fh.read(), f"file {i} ({os.fspath(f)})"
    if isinstance(f, (bytes, bytearray, memoryview)):
        return bytes(f), f"file {i}"
    raise TypeError(f"file {i} must be bytes-like or a path, got {type(f).__name__}")


def parse_png(data: bytes, name: str) -> tuple:
    """(width, height, colour type, IDAT data) of one PNG file.  Checks the signature, IHDR's fields and the CRC of
    every chunk before the first IDAT (as PIL does), and stops at the first chunk after the IDAT run; IDAT data cut off
    by the end of the file is kept as far as it goes (the device then finds the stream truncated)."""
    if data[:8] != SIGNATURE:
        raise ValueError(f"{name}: not a PNG file (signature)")
    pos, idat, ihdr = 8, [], None
    while True:
        if pos + 8 > len(data):
            if idat:
                break
            raise ValueError(f"{name}: truncated before the image data")
        length, typ = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + length]
        if typ == b"IDAT":
            idat.append(body)
        elif idat:
            break
        else:
            if pos + 12 + length > len(data):
                raise ValueError(f"{name}: truncated before the image data (chunk {typ!r})")
            crc = struct.unpack(">I", data[pos + 8 + length:pos + 12 + length])[0]
            if zlib.crc32(typ + body) & 0xFFFFFFFF != crc:
                raise ValueError(f"{name}: CRC of chunk {typ!r} does not match")
            if ihdr is None:
                if typ != b"IHDR" or length != 13:
                    raise ValueError(f"{name}: IHDR: the first chunk must be a 13-byte IHDR, got {typ!r}")
                ihdr = struct.unpack(">IIBBBBB", body)
            elif typ == b"IEND":
                raise ValueError(f"{name}: IDAT: no image data before IEND")
        pos += 12 + length
    w, h, depth, color, comp, filt, interlace = ihdr
    if w == 0 or h == 0 or w > 2**31 - 1 or h > 2**31 - 1:
        raise ValueError(f"{name}: IHDR width/height: {w}x{h} is not a size")
    if depth != 8:
        raise ValueError(f"{name}: IHDR bit depth: {depth}-bit images are not read here (8 only)")
    if color not in (2, 6):
        raise ValueError(f"{name}: IHDR colour type: {COLOR_TYPES.get(color, color)} images are not read here "
                         "(RGB and RGBA only)")
    if comp != 0 or filt != 0:
        raise ValueError(f"{name}: IHDR compression/filter method: {comp}/{filt} (0/0 only)")
    if interlace != 0:
        raise ValueError(f"{name}: IHDR interlace method: interlaced images are not read here")
    return w, h, color, b"".join(idat)


def status_string(status: int) -> str:
    return N.lib().gab200_png_status_string(int(status)).decode()


@torch.no_grad()
def decode_png_status(files, channels: int = 4, device=None) -> tuple:
    """(pixels, statuses, names): decode_png without the raise -- statuses[f] is file f's gab200_png_status (0: ok);
    the pixels of a file with a nonzero status are undefined.  Host-side refusals still raise."""
    if channels not in (3, 4):
        raise ValueError(f"channels must be 3 or 4, got {channels!r}")
    single = isinstance(files, (str, os.PathLike, bytes, bytearray, memoryview))
    items = [files] if single else list(files)
    if not items:
        raise ValueError("decode_png needs at least one file")
    names, idats, colors = [], [], []
    size = None
    for i, f in enumerate(items):
        data, name = _read(f, i)
        w, h, color, idat = parse_png(data, name)
        if size is None:
            size = (w, h)
        elif (w, h) != size:
            raise ValueError(f"{name}: IHDR width/height: {w}x{h}, but file 0 is {size[0]}x{size[1]} (one size per "
                             "call)")
        names.append(name)
        idats.append(idat)
        colors.append(color)
    W, H = size
    F = len(items)
    scratch_bytes = int(N.lib().gab200_png_decode_scratch_bytes(F, H, W))
    if scratch_bytes == 0:
        raise ValueError(f"no PNG decode of {F} files of {W}x{H}")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"decode_png runs on a CUDA device, got {dev}")
    # one pinned buffer: zoff (F int64) | zlen (F int64) | colour types (F bytes, padded to 8) | the IDAT data
    head = 16 * F + (F + 7) // 8 * 8
    lens = [len(d) for d in idats]
    host = torch.empty(head + max(sum(lens), 1), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    offs = np.cumsum([0] + lens[:-1], dtype=np.int64)
    hv[:8 * F].view(np.int64)[:] = offs
    hv[8 * F:16 * F].view(np.int64)[:] = lens
    hv[16 * F:16 * F + F] = colors
    for o, d in zip(offs, idats):
        hv[head + o:head + o + len(d)] = np.frombuffer(d, np.uint8)
    with torch.cuda.device(dev):
        buf = host.to(dev, non_blocking=True)
        scratch_buf = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty((F, H, W, channels), dtype=torch.uint8, device=dev)
        status = torch.empty(F, dtype=torch.int32, device=dev)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        base = buf.data_ptr()
        N.check(N.lib().gab200_png_decode(F, H, W, base + head, base, base + 8 * F, base + 16 * F,
                                          scratch_buf.data_ptr(), out.data_ptr(), channels, status.data_ptr(), stream),
                "gab200_png_decode")
        st = status.tolist()   # the one synchronisation; it also ends the upload out of `host`
    return (out[0] if single else out), st, names


def decode_png(files, channels: int = 4, device=None) -> torch.Tensor:
    """The pixels of one PNG file (bytes-like or a path) as a (H,W,channels) uint8 CUDA tensor, or of a list of F
    files of one size as (F,H,W,channels) -- np.asarray(Image.open(f).convert("RGBA")) bit for bit, its first three
    channels for channels=3.  8-bit RGB or RGBA, not interlaced; anything else raises ValueError naming the file and
    the field.  One upload, one launch, one synchronisation (to read the statuses); a file the device refuses raises
    ValueError naming the first such file and its status."""
    out, st, names = decode_png_status(files, channels, device)
    for i, s in enumerate(st):
        if s != 0:
            raise ValueError(f"{names[i]}: {status_string(s)} (status {s})")
    return out
