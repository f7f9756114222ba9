"""CPU: the H.264 video surface without a launch -- gab200_h264_bound, gab200_h264_scratch_bytes,
gab200_h264_parameter_sets and gab200_h264_encode's refusals against oracle/h264.py, the level table, VideoWriter's
and encode_video's argument checks, and the MP4 muxer's boxes parsed back, co64 included (driven by sample sizes
alone, so no 4 GiB file is written)."""
import ctypes as C
import io
import struct
from fractions import Fraction

import pytest
import torch

from oracle import h264 as O

SIZES = [(2, 2), (16, 16), (18, 34), (32, 2), (2, 32), (176, 144), (550, 802), (1280, 720), (1920, 1080),
         (3840, 2160), (4096, 2304), (8688, 16), (16, 8688)]
REFUSED = [(0, 2), (2, 0), (-2, 2), (3, 2), (2, 3), (4098, 2304), (4096, 2320), (8704, 16), (16, 8704)]


def test_bound_equals_the_oracle():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    for w, h in SIZES:
        assert L.gab200_h264_bound(w, h) == O.bound(w, h) > 0, (w, h)
        assert L.gab200_h264_scratch_bytes(3, h, w) > 0
    for w, h in REFUSED:
        assert L.gab200_h264_bound(w, h) == -1 == O.bound(w, h), (w, h)
        assert L.gab200_h264_scratch_bytes(1, h, w) == 0
    assert L.gab200_h264_scratch_bytes(0, 16, 16) == 0 and L.gab200_h264_scratch_bytes(65536, 16, 16) == 0


def test_level_table():
    from gaussianavatars_b200 import video as V
    assert V.parameter_sets(550, 802, 20, Fraction(25))[0][3] == 31
    assert V.parameter_sets(1920, 1080, 20, Fraction(25))[0][3] == 40
    assert V.parameter_sets(1920, 1080, 20, Fraction(60))[0][3] == 42
    assert V.parameter_sets(176, 144, 20, Fraction(15))[0][3] == 10 and V.parameter_sets(176, 144, 20, Fraction(30))[0][3] == 11
    assert V.parameter_sets(4096, 2304, 20, Fraction(240))[0][3] == 52       # only the rate exceeds every level
    for w, h in SIZES:
        for fps in (Fraction(25), Fraction(30000, 1001), Fraction(60)):
            assert V.parameter_sets(w, h, 20, fps)[0][3] == O.level_idc(w, h, fps), (w, h, fps)


def test_parameter_sets_equal_the_oracle():
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import video as V
    for w, h in SIZES:
        for qp in (0, 26, 51):
            for fps in (Fraction(25), Fraction(30000, 1001), Fraction(1, 2)):
                assert V.parameter_sets(w, h, qp, fps) == O.parameter_sets(w, h, qp, fps.numerator, fps.denominator)
    L = N.lib()
    buf = (C.c_uint8 * 64)()
    assert L.gab200_h264_parameter_sets(16, 16, 20, 25, 1, buf, 8) == -1          # capacity too small
    for bad in ((3, 2, 20, 25, 1), (16, 16, 52, 25, 1), (16, 16, -1, 25, 1), (16, 16, 20, 0, 1), (16, 16, 20, 25, 0)):
        assert L.gab200_h264_parameter_sets(*bad, buf, 64) == -1, bad


def test_encode_refuses_before_any_device_work():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    p, s = 256, 256 * 4
    b = L.gab200_h264_bound(16, 16)
    ok = [1, 16, 16, 20, p, s, p, b, p, None]
    for i, v in [(0, 0), (0, 65536), (1, 3), (2, 0), (3, 52), (3, -1), (4, None), (5, None), (5, s + 16), (6, None),
                 (7, b - 1), (8, None)]:
        args = list(ok)
        args[i] = v
        assert L.gab200_h264_encode(*args) == -1, (i, v)
    assert L.gab200_launch_count() == 0


def test_python_refusals():
    from gaussianavatars_b200 import VideoWriter, encode_video
    good = torch.zeros((2, 32, 48, 3), dtype=torch.uint8)
    with pytest.raises(TypeError):
        encode_video(good.numpy())
    for t, msg in [(good.float(), "uint8"), (good[..., :2], r"\(H, W, 3\)"), (good, "CUDA")]:
        with pytest.raises(ValueError, match=msg):
            encode_video(t)
    for kw, msg in [(dict(qp=52), "qp"), (dict(qp=-1), "qp"), (dict(qp=20.0), "qp"), (dict(fps=25.0), "fps"),
                    (dict(fps=0), "fps"), (dict(fps=Fraction(-1, 2)), "fps"), (dict(batch=0), "batch"),
                    (dict(batch=True), "batch")]:
        with pytest.raises(ValueError, match=msg):
            VideoWriter(io.BytesIO(), 48, 32, **kw)
    for w, h in ((47, 32), (48, 31), (0, 32), (8704, 16)):
        with pytest.raises(ValueError, match="even and positive"):
            VideoWriter(io.BytesIO(), w, h)


def parse(data: bytes, start=0, end=None) -> list:
    """[(type, payload start, payload end, children)] of a box sequence; container boxes are parsed recursively."""
    containers = {b"moov", b"trak", b"mdia", b"minf", b"dinf", b"stbl"}
    out, pos, end = [], start, len(data) if end is None else end
    while pos < end:
        size, kind = struct.unpack(">I4s", data[pos:pos + 8])
        hdr = 8
        if size == 1:
            size = struct.unpack(">Q", data[pos + 8:pos + 16])[0]
            hdr = 16
        assert size >= hdr and pos + size <= end, kind
        kids = parse(data, pos + hdr, pos + size) if kind in containers else []
        out.append((kind, pos + hdr, pos + size, kids))
        pos += size
    return out


def find(tree, path):
    for kind, a, b, kids in tree:
        if kind == path[0]:
            return (kind, a, b, kids) if len(path) == 1 else find(kids, path[1:])
    raise KeyError(path)


def test_muxer_box_tree():
    from gaussianavatars_b200 import video as V
    fps = Fraction(30000, 1001)
    sps, pps = V.parameter_sets(550, 802, 20, fps)
    sizes = [1000, 2345, 77, 4096, 5]
    moov = V.moov_box(sizes, 48, 550, 802, sps, pps, fps)
    assert moov == O.moov(sizes, 48, 550, 802, 20, 30000, 1001)
    tree = parse(moov)
    assert [k for k, *_ in tree] == [b"moov"]
    assert [k for k, *_ in tree[0][3]] == [b"mvhd", b"trak"]
    stbl = find(tree, [b"moov", b"trak", b"mdia", b"minf", b"stbl"])
    assert [k for k, *_ in stbl[3]] == [b"stsd", b"stts", b"stsc", b"stsz", b"stco"]   # no stss: all sync samples
    _, a, b, _ = find(tree, [b"moov", b"trak", b"mdia", b"mdhd"])
    assert struct.unpack(">I", moov[a + 12:a + 16])[0] == 30000 and struct.unpack(">I", moov[a + 16:a + 20])[0] == 5 * 1001
    _, a, b, _ = find(stbl[3], [b"stts"])
    assert struct.unpack(">IIII", moov[a:b]) == (0, 1, 5, 1001)
    _, a, b, _ = find(stbl[3], [b"stsz"])
    assert struct.unpack(">III5I", moov[a:b]) == (0, 0, 5, *sizes)
    _, a, b, _ = find(stbl[3], [b"stco"])
    assert list(struct.unpack(">5I", moov[a + 8:b])) == [48, 1048, 3393, 3470, 7566]
    _, a, b, _ = find(stbl[3], [b"stsd"])
    avcc = moov.index(b"avcC")
    assert moov[avcc + 4:avcc + 10] == bytes([1, 66, 0xC0, 31, 0xFF, 0xE1])
    assert moov[avcc + 10:avcc + 12] == struct.pack(">H", len(sps)) and moov[avcc + 12:avcc + 12 + len(sps)] == sps
    _, a, b, _ = find(tree, [b"moov", b"trak", b"tkhd"])
    assert struct.unpack(">II", moov[b - 8:b]) == (550 << 16, 802 << 16)
    # a whole file: ftyp | mdat (64-bit largesize) | moov
    samples = [bytes([0, 0, 0, 4, 0x65, 0x88, 0x82, 0x80])] * 3
    data = O.mp4(samples, 16, 16, 20)
    top = parse(data)
    assert [k for k, *_ in top] == [b"ftyp", b"mdat", b"moov"]
    assert data[top[1][1]:top[1][2]] == samples[0] + bytes([0, 0, 0, 4, 0x65, 0x88, 0x83, 0x80]) + samples[0]


def test_co64_from_sample_sizes_alone():
    from gaussianavatars_b200 import video as V
    sps, pps = V.parameter_sets(1920, 1080, 20, Fraction(25))
    sizes = [2 ** 31, 2 ** 31 - 16, 16, 12345]
    moov = V.moov_box(sizes, 48, 1920, 1080, sps, pps, Fraction(25))
    assert moov == O.moov(sizes, 48, 1920, 1080, 20, 25, 1)
    stbl = find(parse(moov), [b"moov", b"trak", b"mdia", b"minf", b"stbl"])
    assert [k for k, *_ in stbl[3]][-1] == b"co64"
    _, a, b, _ = find(stbl[3], [b"co64"])
    assert struct.unpack(">I4Q", moov[a + 4:b]) == (4, 48, 48 + 2 ** 31, 48 + 2 ** 32 - 16, 48 + 2 ** 32)
    small = V.moov_box(sizes[:2], 48, 1920, 1080, sps, pps, Fraction(25))
    assert b"stco" in small and b"co64" not in small      # the last offset is below 2^32
