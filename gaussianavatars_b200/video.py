"""MP4 videos written from device frames: what render.py's `ffmpeg -framerate 25 -i '<dir>/*.png' -pix_fmt yuv420p
renders.mp4` makes of the PNG files it wrote, without the PNG files.

    with VideoWriter(path, W, H, fps=25, qp=20, gop=25) as vw:   # render.py's renders.mp4 / gt.mp4 / renders_mesh.mp4
        for t in timesteps:
            player.run(...)
            vw.add(player.display)                        # CUDA (H,W,3) or (K,H,W,3) uint8
    data = encode_video(frames, fps=25, qp=20, gop=1, deblock=False, intra4x4=False)   # a whole MP4 in memory

The frames are encoded on the device (csrc/h264.cu, include/gab200_rasterizer.h gab200_h264_encode and
gab200_h264_encode_stream): H.264 Constrained Baseline, one fixed QP, BT.601 limited-range 4:2:0.  With gop=1 (the
default) every frame is an IDR picture; with gop=N every N-th frame is, and the others are P pictures that refer to
the frame before them, which is far smaller when successive frames look alike (a fixed camera).  Deblocking is off by
default, so a decoder outputs the encoder's reconstruction as it is; with deblock=True every slice turns the in-loop
deblocking filter on, and the encoder filters each picture as a decoder does (gab200_h264_encode_deblocked), the P
pictures predicting from the filtered one.  With intra4x4=True an intra macroblock may also be I_NxN, nine
directional predictions per 4x4 block in place of one per 16x16 block (gab200_h264_encode_flags); the parameter sets
are the same, so every decoder that plays the other files plays these.  Only the compressed samples cross to the host, through a ring of pinned
slots; the file is ftyp | mdat | moov, muxed here, with an stss box listing the IDR frames when gop > 1.  The bytes are
deterministic and differ from libx264's.
"""
from __future__ import annotations

import ctypes as C
import io
import os
import struct
from collections import deque
from fractions import Fraction

import torch

from . import _native as N
from .png import launch_copy

MAX_QP = 51
H264_DEBLOCK = 1          # include/gab200_rasterizer.h GAB200_H264_DEBLOCK
H264_INTRA4X4 = 2         # GAB200_H264_INTRA4X4


def video_bound(width: int, height: int) -> int:
    """The largest sample of one width x height frame (gab200_h264_bound); raises for a size no stream can hold."""
    b = int(N.lib().gab200_h264_bound(int(width), int(height)))
    if b < 0:
        raise ValueError(f"no H.264 video of {width}x{height}: width and height must be even and positive, and the "
                         "frame at most 36864 macroblocks with sides of at most 543 (level 5.2)")
    return b


def slot_stride(width: int, height: int, gop: int = 1) -> int:
    """Bytes per sample in an output buffer: the bound (of a P sample when gop > 1) rounded up to 16 (gab200_png_copy
    moves 16-byte words)."""
    b = video_bound(width, height)
    if gop > 1:
        b = int(N.lib().gab200_h264_p_bound(int(width), int(height)))
    return (b + 15) // 16 * 16


def _check_gop(gop) -> int:
    if isinstance(gop, bool) or not isinstance(gop, int) or not 1 <= gop <= 65535:
        raise ValueError(f"gop must be an int in 1..65535, got {gop!r}")
    return gop


def _check_deblock(deblock) -> bool:
    if not isinstance(deblock, bool):
        raise ValueError(f"deblock must be a bool, got {deblock!r}")
    return deblock


def _check_intra4x4(intra4x4) -> bool:
    if not isinstance(intra4x4, bool):
        raise ValueError(f"intra4x4 must be a bool, got {intra4x4!r}")
    return intra4x4


def _check_qp(qp) -> int:
    if isinstance(qp, bool) or not isinstance(qp, int) or not 0 <= qp <= MAX_QP:
        raise ValueError(f"qp must be an int in 0..{MAX_QP}, got {qp!r}")
    return qp


def _check_fps(fps) -> Fraction:
    if isinstance(fps, bool) or not isinstance(fps, (int, Fraction)):
        raise ValueError(f"fps must be an int or a fractions.Fraction, got {fps!r}")
    fps = Fraction(fps)
    if fps <= 0 or fps.numerator > 2 ** 30 or fps.denominator > 2 ** 31 - 1:
        raise ValueError(f"fps must be positive with a numerator up to 2^30, got {fps}")
    return fps


def check_frames(frames, name: str = "frames") -> tuple:
    """(K, H, W) of a CUDA uint8 (H,W,3) or (K,H,W,3) contiguous tensor; raises naming what is wrong."""
    if not isinstance(frames, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(frames).__name__}")
    if frames.dtype != torch.uint8:
        raise ValueError(f"{name} must be uint8 (display bytes), got {frames.dtype}")
    if frames.dim() not in (3, 4) or frames.shape[-1] != 3:
        raise ValueError(f"{name} must be (H, W, 3) or (K, H, W, 3), got shape {tuple(frames.shape)}")
    if frames.device.type != "cuda":
        raise ValueError(f"{name} must be on a CUDA device (the encode runs there), got {frames.device}")
    if not frames.is_contiguous():
        raise ValueError(f"{name} must be contiguous (rows of 3W bytes); call .contiguous() first")
    K = 1 if frames.dim() == 3 else int(frames.shape[0])
    H, W = int(frames.shape[-3]), int(frames.shape[-2])
    if K < 1:
        raise ValueError(f"{name} must hold at least one frame, got shape {tuple(frames.shape)}")
    video_bound(W, H)
    return K, H, W


def parameter_sets(width: int, height: int, qp: int, fps: Fraction, gop: int = 1) -> tuple:
    """(SPS, PPS) NAL units of the stream (gab200_h264_stream_parameter_sets)."""
    buf = (C.c_uint8 * 256)()
    n = int(N.lib().gab200_h264_stream_parameter_sets(width, height, qp, fps.numerator, fps.denominator, gop, buf,
                                                      len(buf)))
    if n < 0:
        raise ValueError(f"no parameter sets for {width}x{height} at qp {qp}, {fps} frames/s")
    data = bytes(buf[:n])
    ls = struct.unpack(">H", data[:2])[0]
    sps = data[2:2 + ls]
    lp = struct.unpack(">H", data[2 + ls:4 + ls])[0]
    return sps, data[4 + ls:4 + ls + lp]


def launch_encode(frames: torch.Tensor, qp: int, scratch_buf: torch.Tensor, out: torch.Tensor, out_len: torch.Tensor):
    """Enqueues gab200_h264_encode on the current stream: frames (K,H,W,3) -> sample k in out[k] ((>= K, stride)
    uint8), its length in out_len[k] (int64).  Reads nothing on the host: capturable."""
    K, H, W = check_frames(frames)
    stream = C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)
    N.check(N.lib().gab200_h264_encode(K, H, W, qp, frames.data_ptr(), scratch_buf.data_ptr(), out.data_ptr(),
                                       out.stride(0), out_len.data_ptr(), stream), "gab200_h264_encode")


def launch_encode_stream(frames: torch.Tensor, qp: int, gop: int, state: torch.Tensor, scratch_buf: torch.Tensor,
                         out: torch.Tensor, out_len: torch.Tensor):
    """Enqueues gab200_h264_encode_stream on the current stream: frames (K,H,W,3) are the next K frames of the stream
    whose state (state_buffer) the encode reads and advances on the device.  Reads nothing on the host: capturable."""
    K, H, W = check_frames(frames)
    stream = C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)
    N.check(N.lib().gab200_h264_encode_stream(K, H, W, qp, gop, frames.data_ptr(), state.data_ptr(),
                                              scratch_buf.data_ptr(), out.data_ptr(), out.stride(0),
                                              out_len.data_ptr(), stream), "gab200_h264_encode_stream")


def launch_encode_deblocked(frames: torch.Tensor, qp: int, gop: int, state, scratch_buf: torch.Tensor,
                            out: torch.Tensor, out_len: torch.Tensor):
    """Enqueues gab200_h264_encode_deblocked on the current stream: launch_encode_stream's samples with the deblocking
    filter on, scratch from deblocked_scratch.  state may be None when gop is 1.  Reads nothing on the host:
    capturable."""
    K, H, W = check_frames(frames)
    stream = C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)
    N.check(N.lib().gab200_h264_encode_deblocked(K, H, W, qp, gop, frames.data_ptr(),
                                                 None if state is None else state.data_ptr(), scratch_buf.data_ptr(),
                                                 out.data_ptr(), out.stride(0), out_len.data_ptr(), stream),
            "gab200_h264_encode_deblocked")


def launch_encode_flags(frames: torch.Tensor, qp: int, gop: int, deblock: bool, intra4x4: bool, state, scratch_buf,
                        out: torch.Tensor, out_len: torch.Tensor):
    """Enqueues gab200_h264_encode_flags on the current stream: launch_encode_deblocked's samples (the filter only
    when deblock) with I_NxN macroblocks when intra4x4, scratch from flags_scratch.  state may be None when gop is 1.
    Reads nothing on the host: capturable."""
    K, H, W = check_frames(frames)
    stream = C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)
    N.check(N.lib().gab200_h264_encode_flags(K, H, W, qp, gop, _flags(deblock, intra4x4), frames.data_ptr(),
                                             None if state is None else state.data_ptr(), scratch_buf.data_ptr(),
                                             out.data_ptr(), out.stride(0), out_len.data_ptr(), stream),
            "gab200_h264_encode_flags")


def _flags(deblock: bool, intra4x4: bool) -> int:
    return (H264_DEBLOCK if deblock else 0) | (H264_INTRA4X4 if intra4x4 else 0)


def state_buffer(H: int, W: int, device) -> torch.Tensor:
    """A zeroed stream state: its next frame is an IDR picture."""
    n = int(N.lib().gab200_h264_state_bytes(H, W))
    if n == 0:
        raise ValueError(f"no H.264 stream of {W}x{H}")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def scratch(K: int, H: int, W: int, device) -> torch.Tensor:
    n = int(N.lib().gab200_h264_scratch_bytes(K, H, W))
    if n == 0:
        raise ValueError(f"no H.264 encode of {K} frames of {W}x{H}")
    return torch.empty(n, dtype=torch.uint8, device=device)


def deblocked_scratch(K: int, H: int, W: int, gop: int, device) -> torch.Tensor:
    n = int(N.lib().gab200_h264_deblocked_scratch_bytes(K, H, W, gop))
    if n == 0:
        raise ValueError(f"no deblocked H.264 encode of {K} frames of {W}x{H} with gop {gop}")
    return torch.empty(n, dtype=torch.uint8, device=device)


def flags_scratch(K: int, H: int, W: int, gop: int, deblock: bool, intra4x4: bool, device) -> torch.Tensor:
    n = int(N.lib().gab200_h264_flags_scratch_bytes(K, H, W, gop, _flags(deblock, intra4x4)))
    if n == 0:
        raise ValueError(f"no H.264 encode of {K} frames of {W}x{H} with gop {gop}")
    return torch.empty(n, dtype=torch.uint8, device=device)


# ---- MP4 ---------------------------------------------------------------------------------------------------------
def _box(kind: bytes, *payload: bytes) -> bytes:
    body = b"".join(payload)
    return struct.pack(">I", 8 + len(body)) + kind + body


def _full(kind: bytes, version: int, flags: int, *payload: bytes) -> bytes:
    return _box(kind, struct.pack(">I", (version << 24) | flags), *payload)


_MATRIX = struct.pack(">9I", 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)
FTYP = _box(b"ftyp", b"isom", struct.pack(">I", 512), b"isomiso2avc1mp41")
MDAT_HEADER = 16          # size 1, 'mdat', 64-bit largesize


def moov_box(sizes, first_offset: int, width: int, height: int, sps: bytes, pps: bytes, fps: Fraction,
             sync=None) -> bytes:
    """The movie box of one video track whose samples of `sizes` bytes lie back to back from file offset
    `first_offset`, one chunk per sample (stco, or co64 once an offset passes 2^32).  sync: None when every sample is
    a sync sample (no stss), else the 1-based numbers of the sync samples, listed in an stss box."""
    n = len(sizes)
    dur = n * fps.denominator
    avcc = _box(b"avcC", bytes([1, sps[1], sps[2], sps[3], 0xFF, 0xE1]), struct.pack(">H", len(sps)), sps, bytes([1]),
                struct.pack(">H", len(pps)), pps)
    avc1 = _box(b"avc1", bytes(6), struct.pack(">H", 1), bytes(16), struct.pack(">HH", width, height),
                struct.pack(">II", 0x480000, 0x480000), bytes(4), struct.pack(">H", 1), bytes(32),
                struct.pack(">Hh", 0x18, -1), avcc)
    offs, o = [], first_offset
    for s in sizes:
        offs.append(o)
        o += int(s)
    if offs and offs[-1] >= 2 ** 32:
        co = _full(b"co64", 0, 0, struct.pack(">I", n), struct.pack(">%dQ" % n, *offs))
    else:
        co = _full(b"stco", 0, 0, struct.pack(">I", n), struct.pack(">%dI" % n, *offs))
    stts = struct.pack(">III", 1, n, fps.denominator) if n else struct.pack(">I", 0)
    stbl = _box(b"stbl", _full(b"stsd", 0, 0, struct.pack(">I", 1), avc1), _full(b"stts", 0, 0, stts),
                _full(b"stsc", 0, 0, struct.pack(">IIII", 1, 1, 1, 1)),
                _full(b"stsz", 0, 0, struct.pack(">II", 0, n), struct.pack(">%dI" % n, *sizes)),
                b"" if sync is None else _full(b"stss", 0, 0, struct.pack(">I", len(sync)),
                                               struct.pack(">%dI" % len(sync), *sync)), co)
    minf = _box(b"minf", _full(b"vmhd", 0, 1, bytes(8)),
                _box(b"dinf", _full(b"dref", 0, 0, struct.pack(">I", 1), _full(b"url ", 0, 1))), stbl)
    mdia = _box(b"mdia", _full(b"mdhd", 0, 0, struct.pack(">IIIIHH", 0, 0, fps.numerator, dur, 0x55C4, 0)),
                _full(b"hdlr", 0, 0, bytes(4), b"vide", bytes(12), b"VideoHandler\x00"), minf)
    tkhd = _full(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, 1, 0, dur), bytes(8), struct.pack(">hhHH", 0, 0, 0, 0),
                 _MATRIX, struct.pack(">II", width << 16, height << 16))
    mvhd = _full(b"mvhd", 0, 0, struct.pack(">IIII", 0, 0, fps.numerator, dur), struct.pack(">IH", 0x10000, 0x100),
                 bytes(10), _MATRIX, bytes(24), struct.pack(">I", 2))
    return _box(b"moov", mvhd, _box(b"trak", tkhd, mdia))


class VideoWriter:
    """An MP4 file of H.264 frames encoded on the device.  add() copies frames device to device into the current
    batch; a full batch is encoded on the current stream and its samples copied to a ring of pinned host slots.  add()
    waits on the GPU only when the ring is full; close() encodes the partial last batch and writes the moov box.

    path: a file name, or a seekable binary file object (left open).  fps: an int or a fractions.Fraction (the
    track's timescale is its numerator, each sample lasts its denominator).  gop: every gop-th frame, the first
    included, is an IDR picture and the others P pictures (1: every frame an IDR picture); the writer owns the
    stream's state on the device, so a batch may start anywhere in a GOP.  deblock: the in-loop deblocking filter on
    in every slice of the stream (a bool; the writer keeps one mode for its whole stream).  intra4x4: intra
    macroblocks may also be I_NxN, each 4x4 block predicted on its own (a bool, for the whole stream)."""

    RING = 3

    def __init__(self, path, width: int, height: int, fps=25, qp: int = 20, batch: int = 16, device=None, gop: int = 1,
                 deblock: bool = False, intra4x4: bool = False):
        self.fps = _check_fps(fps)
        self.qp = _check_qp(qp)
        self.gop = _check_gop(gop)
        self.deblock = _check_deblock(deblock)
        self.intra4x4 = _check_intra4x4(intra4x4)
        if isinstance(batch, bool) or not isinstance(batch, int) or not 1 <= batch <= 65535:
            raise ValueError(f"batch must be an int in 1..65535, got {batch!r}")
        self.W, self.H = int(width), int(height)
        self.stride = slot_stride(self.W, self.H, self.gop)
        self.sps, self.pps = parameter_sets(self.W, self.H, self.qp, self.fps, self.gop)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"VideoWriter encodes on a CUDA device, got {self.device}")
        self.batch = batch
        with torch.cuda.device(self.device):
            self._frames = torch.empty((batch, self.H, self.W, 3), dtype=torch.uint8, device=self.device)
            if self.intra4x4:
                self._scratch = flags_scratch(batch, self.H, self.W, self.gop, self.deblock, True, self.device)
            elif self.deblock:
                self._scratch = deblocked_scratch(batch, self.H, self.W, self.gop, self.device)
            else:
                self._scratch = scratch(batch, self.H, self.W, self.device)
            self._out = torch.empty((batch, self.stride), dtype=torch.uint8, device=self.device)
            self._out_len = torch.empty(batch, dtype=torch.int64, device=self.device)
            self._state = state_buffer(self.H, self.W, self.device) if self.gop > 1 else None
            self._ring = [(torch.empty((batch, self.stride), dtype=torch.uint8, pin_memory=True),
                           torch.empty(batch, dtype=torch.int64, pin_memory=True)) for _ in range(self.RING)]
        self._pending = deque()        # (ring slot, event, frame count), oldest first
        self._next_slot = 0
        self._fill = 0
        self._sizes = []
        self._sync = []                # 1-based numbers of the IDR samples
        self._own = isinstance(path, (str, os.PathLike))
        self._f = open(path, "wb") if self._own else path
        self._start = self._f.tell()
        self._f.write(FTYP)
        self._mdat = self._f.tell()
        self._f.write(struct.pack(">I4sQ", 1, b"mdat", MDAT_HEADER))
        self.closed = False

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def add(self, frames: torch.Tensor):
        """Append one (H,W,3) frame or a (K,H,W,3) batch: CUDA uint8, contiguous, of the writer's size."""
        if self.closed:
            raise ValueError("add() on a closed VideoWriter")
        K, H, W = check_frames(frames)
        if (W, H) != (self.W, self.H):
            raise ValueError(f"frames are {W}x{H}, but the writer is {self.W}x{self.H}")
        if frames.device != self.device:
            raise ValueError(f"frames are on {frames.device}, but the writer encodes on {self.device}")
        src = frames.view(K, H, W, 3)
        i = 0
        with torch.cuda.device(self.device):
            while i < K:
                n = min(K - i, self.batch - self._fill)
                self._frames[self._fill:self._fill + n].copy_(src[i:i + n])
                self._fill += n
                i += n
                if self._fill == self.batch:
                    self._encode()

    def _encode(self):
        n, self._fill = self._fill, 0
        slot = self._next_slot
        self._next_slot = (slot + 1) % self.RING
        if len(self._pending) == self.RING:
            self._drain(1)
        if self.intra4x4:
            launch_encode_flags(self._frames[:n], self.qp, self.gop, self.deblock, True, self._state, self._scratch,
                                self._out, self._out_len)
        elif self.deblock:
            launch_encode_deblocked(self._frames[:n], self.qp, self.gop, self._state, self._scratch, self._out,
                                    self._out_len)
        elif self._state is None:
            launch_encode(self._frames[:n], self.qp, self._scratch, self._out, self._out_len)
        else:
            launch_encode_stream(self._frames[:n], self.qp, self.gop, self._state, self._scratch, self._out,
                                 self._out_len)
        host, host_len = self._ring[slot]
        launch_copy(self._out[:n], self._out_len[:n], host, host_len)
        ev = torch.cuda.Event()
        ev.record()
        self._pending.append((slot, ev, n))

    def _drain(self, count: int):
        for _ in range(count):
            slot, ev, n = self._pending.popleft()
            ev.synchronize()
            host, host_len = self._ring[slot]
            lens = host_len[:n].tolist()
            hv = host.numpy()
            for k in range(n):
                s = bytearray(hv[k, :lens[k]].tobytes())
                if s[4] == 0x65:                   # an IDR picture
                    if len(self._sync) % 2:
                        s[6] |= 1                  # idr_pic_id 2 on odd IDR pictures (include/gab200_rasterizer.h)
                    self._sync.append(len(self._sizes) + 1)
                self._f.write(s)
                self._sizes.append(lens[k])

    def close(self):
        if self.closed:
            return
        with torch.cuda.device(self.device):
            if self._fill:
                self._encode()
            self._drain(len(self._pending))
        end = self._f.tell()
        self._f.write(moov_box(self._sizes, self._mdat + MDAT_HEADER, self.W, self.H, self.sps, self.pps, self.fps,
                               self._sync if self.gop > 1 else None))
        after = self._f.tell()
        self._f.seek(self._mdat + 8)
        self._f.write(struct.pack(">Q", end - self._mdat))
        self._f.seek(after)
        if self._own:
            self._f.close()
        self.closed = True

    @property
    def frames_written(self) -> int:
        return len(self._sizes)


@torch.no_grad()
def encode_video(frames: torch.Tensor, fps=25, qp: int = 20, gop: int = 1, deblock: bool = False,
                 intra4x4: bool = False) -> bytes:
    """A whole MP4 of a CUDA uint8 (H,W,3) frame or (K,H,W,3) clip, in memory."""
    _check_intra4x4(intra4x4)
    K, H, W = check_frames(frames)
    buf = io.BytesIO()
    with VideoWriter(buf, W, H, fps=fps, qp=qp, batch=min(K, 16), device=frames.device, gop=gop,
                     deblock=deblock, intra4x4=intra4x4) as vw:
        vw.add(frames)
    return buf.getvalue()
