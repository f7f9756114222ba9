"""The training frames held on the device: a tile-packed lossless frame store, decoded inside the captured iteration.

    store = FrameStore(width, height, bg, device)
    ids = store.add_rgba(rgba_u8)               # decoded capture frames (K,H,W,4): composite + encode, once
    ids = store.add_png(paths)                  # or the capture's PNG files, decoded on the device
    ids = store.add_png(paths, resize=True)     # ... of another size: composited, then resized as the loader does
    gt, mask = store.decode(ids)                # eager: the bytes composite_rgba made, bit for bit
    frame = GraphedFrame(pc, width, height, fovx, fovy, bg, frames=store)
    frame.set_inputs(cameras=..., timestep=t, frames=ids)   # K ints: the replay decodes them on the device

A frame is four uint8 planes -- R, G, B of the composited ground truth (what GraphedFrame.gt holds) and M, the alpha
bytes (GraphedFrame.mask; 255 for a frame added without a mask) -- coded per 16x16 tile and plane as a base byte and
zigzagged mod-256 2-D differences packed at the tile's own bit width (include/gab200_rasterizer.h,
gab200_frame_encode_plan; oracle/frame_codec.py restates it).  Transparent regions composite to the constant background
and cost 8 bytes per tile; no frame takes more than n_tiles * 1036 + 8 bytes, 1036/1024 of the frame rounded up
to whole tiles.

The encoded frames live in one device arena with a device index (an int64 byte offset per frame, a uint32 offset per
tile).  `add` encodes a batch on the device and may synchronise to learn its size: growing the arena reallocates and
copies it, so a captured frame that reads the store re-captures on its next run().  Setup time only.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _native as N
from .png import decode_png
from .training import composite_rgba

TILE = 16
RECORD_MAX = 8 + 32 * 8 * 4   # bytes of one tile's record at width 8 in every plane
PNG_BATCH = 256               # files per decode in add_png (the fastest of 16, 64, 256: profiles/h100/png_decode.jsonl)


def _tiles(height: int, width: int) -> int:
    return ((height + TILE - 1) // TILE) * ((width + TILE - 1) // TILE)


def _grow(t: torch.Tensor, used: int, need: int) -> torch.Tensor:
    """t if it holds `need` elements, else a tensor of twice that many holding t's first `used`."""
    if t.numel() >= need:
        return t
    out = torch.empty(max(need, 2 * t.numel()), dtype=t.dtype, device=t.device)
    out[:used].copy_(t[:used])
    return out


class FrameStore:
    def __init__(self, width: int, height: int, bg, device=None):
        """width x height frames composited over `bg` (3 values; the background the frames' ground truth was, or will
        be in add_rgba, composited with)."""
        self.W, self.H = int(width), int(height)
        if self.W <= 0 or self.H <= 0:
            raise ValueError(f"a frame store holds frames of a positive size, got {self.W}x{self.H}")
        b = torch.as_tensor(bg, dtype=torch.float32).reshape(-1)
        if b.numel() != 3:
            raise ValueError(f"bg must hold 3 values, got {b.numel()}")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: a FrameStore lives on a CUDA device")
        self.bg = b.to(self.device).contiguous()
        self.n_tiles = _tiles(self.H, self.W)
        self._n = 0          # frames
        self._used = 0       # arena bytes
        self.arena = torch.empty(0, dtype=torch.uint8, device=self.device)
        self.frame_base = torch.empty(0, dtype=torch.int64, device=self.device)
        self.tile_off = torch.empty(0, dtype=torch.int32, device=self.device)   # uint32 in the ABI (< 2^31 here)

    # ---- size ------------------------------------------------------------------------------------------------------
    def __len__(self) -> int:
        return self._n

    @property
    def nbytes(self) -> int:
        """Bytes the stored frames take on the device: their records and their index."""
        return self._used + self._n * (8 + 4 * self.n_tiles)

    @property
    def raw_nbytes(self) -> int:
        """The same frames held raw: 4 bytes per pixel (R, G, B, mask)."""
        return self._n * 4 * self.H * self.W

    def pointers(self) -> tuple:
        """The addresses a decode reads (the arena and its index): they change only when the store grows."""
        return (self.arena.data_ptr(), self.frame_base.data_ptr(), self.tile_off.data_ptr())

    # ---- adding frames ---------------------------------------------------------------------------------------------
    def _batch(self, t, name, channels):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() not in (3, 4) or \
                tuple(t.shape[-3:]) != (channels, self.H, self.W):
            raise ValueError(f"{name} must be a uint8 ({channels}, {self.H}, {self.W}) or (F, {channels}, {self.H}, "
                             f"{self.W}) tensor, got {getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
        t = t if t.dim() == 4 else t.unsqueeze(0)
        return t.to(self.device).contiguous()

    @torch.no_grad()
    def add(self, gt_u8: torch.Tensor, mask_u8: Optional[torch.Tensor] = None) -> list:
        """Encodes one frame ((3,H,W) ground truth, (1,H,W) mask) or a batch ((F,3,H,W), (F,1,H,W)) on the device and
        returns the new frames' ids.  mask None: M = 255.  Synchronises once to learn the encoded size."""
        gt = self._batch(gt_u8, "gt_u8", 3)
        mask = None if mask_u8 is None else self._batch(mask_u8, "mask_u8", 1)
        if mask is not None and mask.shape[0] != gt.shape[0]:
            raise ValueError(f"mask_u8 holds {mask.shape[0]} frames, gt_u8 {gt.shape[0]}")
        F, T, dev = int(gt.shape[0]), self.n_tiles, self.device
        if F == 0:
            return []
        L = N.lib()
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            units = torch.empty((F, T), dtype=torch.int32, device=dev)
            N.check(L.gab200_frame_encode_plan(F, self.H, self.W, gt.data_ptr(), N.ptr(mask), units.data_ptr(),
                                               stream), "gab200_frame_encode_plan")
            ends = units.to(torch.int64).cumsum(1)
            tile_off = (ends - units).to(torch.int32)            # exclusive scan per frame, 8-byte units
            sizes = ends[:, -1] * 8                              # bytes per frame
            frame_base = self._used + sizes.cumsum(0) - sizes
            total = int(sizes.sum())                             # the one synchronisation
            self.arena = _grow(self.arena, self._used, self._used + total)
            self.frame_base = _grow(self.frame_base, self._n, self._n + F)
            self.tile_off = _grow(self.tile_off, self._n * T, (self._n + F) * T)
            self.frame_base[self._n:self._n + F].copy_(frame_base)
            self.tile_off[self._n * T:(self._n + F) * T].copy_(tile_off.reshape(-1))
            N.check(L.gab200_frame_encode(F, self.H, self.W, gt.data_ptr(), N.ptr(mask),
                                          self.frame_base[self._n:].data_ptr(), self.tile_off[self._n * T:].data_ptr(),
                                          self.arena.data_ptr(), stream), "gab200_frame_encode")
        ids = list(range(self._n, self._n + F))
        self._n += F
        self._used += total
        return ids

    def add_rgba(self, rgba_u8: torch.Tensor, resize: bool = False) -> list:
        """Decoded capture frames ((H,W,4) or (F,H,W,4) uint8) -> training.composite_rgba onto the store's background,
        then add(gt, mask).  A CPU batch is uploaded first.  resize: frames of another size are composited at their
        own size, then resized to the store's (composite_rgba(size=): the reference loader's bicubic resize, and the
        alpha bytes resized as an "L" image); without it they must have the store's size."""
        if isinstance(rgba_u8, torch.Tensor) and rgba_u8.device.type == "cpu":
            rgba_u8 = rgba_u8.to(self.device)
        gt, mask = composite_rgba(rgba_u8, self.bg, size=(self.W, self.H) if resize else None)
        return self.add(gt, mask)

    def add_png(self, files, batch: int = PNG_BATCH, resize: bool = False) -> list:
        """The capture's PNG frames (paths or bytes; RGB or RGBA, the store's size) decoded on the device
        (png.decode_png) `batch` files at a time, each batch then add_rgba'd; returns the new frames' ids.  The stored
        frames are those of PIL's convert("RGBA") + add_rgba byte for byte.  `batch` bounds the decode's device memory:
        about 2 H (4W + 1) bytes per file.

        resize: the files may have another size than the store's (one size per batch): each batch is decoded,
        composited at its own size and resized to the store's -- what the reference's loader makes of a capture
        larger than its camera (resize.loader_size), byte for byte.  Without it a file of another size raises."""
        if isinstance(batch, bool) or not isinstance(batch, int) or batch < 1:
            raise ValueError(f"batch must be a positive int, got {batch!r}")
        files = list(files)
        ids = []
        for i in range(0, len(files), batch):
            rgba = decode_png(files[i:i + batch], 4, self.device)
            if not resize and tuple(rgba.shape[1:3]) != (self.H, self.W):
                raise ValueError(f"files {i}..{i + len(rgba) - 1} are {rgba.shape[2]}x{rgba.shape[1]}, the store holds "
                                 f"{self.W}x{self.H} frames (resize=True resizes them)")
            ids += self.add_rgba(rgba, resize)
        return ids

    # ---- reading frames --------------------------------------------------------------------------------------------
    def check_ids(self, ids) -> list:
        """ids as a list of host ints, each checked against the number of stored frames (the decode reads them
        unchecked on the device)."""
        if isinstance(ids, torch.Tensor):
            ids = ids.reshape(-1).tolist()
        elif isinstance(ids, int):   # a bool is refused below
            ids = [ids]
        out = []
        for i in ids:
            if isinstance(i, bool) or not isinstance(i, int) or not 0 <= i < self._n:
                raise ValueError(f"frame ids index the store's {self._n} frames: got {i!r}")
            out.append(int(i))
        return out

    def launch_decode(self, ids_dev: torch.Tensor, gt_out: torch.Tensor, mask_out: Optional[torch.Tensor] = None):
        """Enqueues gab200_frame_decode on the current stream: frames ids_dev ((K,) device int32, read on the device)
        -> gt_out (K,3,H,W) and mask_out (K,1,H,W) (None: not written), or (3,H,W) / (1,H,W) for K = 1.
        Capturable: it reads nothing on the host."""
        K = int(ids_dev.numel())
        lead = () if gt_out.dim() == 3 else (K,)
        if ids_dev.dtype != torch.int32 or ids_dev.device != self.device or not ids_dev.is_contiguous():
            raise ValueError(f"frame ids must be a contiguous int32 tensor on {self.device}")
        if lead == () and K != 1:
            raise ValueError(f"a (3, H, W) output holds one frame, got {K} ids")
        for t, n, c in ((gt_out, "gt_out", 3), (mask_out, "mask_out", 1)):
            if t is not None and (t.dtype != torch.uint8 or tuple(t.shape) != lead + (c, self.H, self.W) or
                                  t.device != self.device or not t.is_contiguous()):
                raise ValueError(f"{n} must be a contiguous uint8 {lead + (c, self.H, self.W)} tensor on {self.device}")
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            N.check(N.lib().gab200_frame_decode(K, self.H, self.W, ids_dev.data_ptr(), self.arena.data_ptr(),
                                                self.frame_base.data_ptr(), self.tile_off.data_ptr(),
                                                gt_out.data_ptr(), N.ptr(mask_out), C.c_void_p(stream)),
                    "gab200_frame_decode")
        return gt_out, mask_out

    @torch.no_grad()
    def decode(self, ids) -> tuple:
        """(gt (K,3,H,W), mask (K,1,H,W)) uint8 of frames `ids` (an int or K ints), decoded on the device."""
        ids = self.check_ids(ids)
        dev = self.device
        idt = torch.tensor(ids, dtype=torch.int32).to(dev)
        gt = torch.empty((len(ids), 3, self.H, self.W), dtype=torch.uint8, device=dev)
        mask = torch.empty((len(ids), 1, self.H, self.W), dtype=torch.uint8, device=dev)
        return self.launch_decode(idt, gt, mask)
