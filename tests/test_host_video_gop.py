"""CPU: the H.264 stream surface without a launch -- gab200_h264_p_bound, gab200_h264_state_bytes,
gab200_h264_stream_scratch_bytes and gab200_h264_stream_parameter_sets against tests/h264_stream_oracle.py, the
refusals of gab200_h264_encode_stream and VideoWriter(gop=), and the muxer's stss box."""
import ctypes as C
import struct
from fractions import Fraction

import pytest

from oracle import h264 as O
from tests import h264_stream_oracle as S


@pytest.fixture(scope="module")
def L():
    from gaussianavatars_b200 import _native as N
    return N.lib()


SIZES = [(2, 2), (16, 16), (18, 34), (550, 802), (1920, 1080), (8688, 16)]


def test_p_bound_state_and_scratch_sizes_agree_with_the_oracle(L):
    for w, h in SIZES:
        assert L.gab200_h264_p_bound(w, h) == S.p_bound(w, h) > L.gab200_h264_bound(w, h), (w, h)
        nmb = ((w + 15) // 16) * ((h + 15) // 16)
        assert L.gab200_h264_state_bytes(h, w) == 256 + (384 * nmb + 255) // 256 * 256
        assert L.gab200_h264_stream_scratch_bytes(3, h, w, 25) == L.gab200_h264_scratch_bytes(3, h, w) > 0
    for w, h in [(3, 2), (0, 16), (16, 8704 * 16)]:
        assert L.gab200_h264_p_bound(w, h) == -1 == S.p_bound(w, h)
        assert L.gab200_h264_state_bytes(h, w) == 0
    for gop in (0, 65536, -1):
        assert L.gab200_h264_stream_scratch_bytes(1, 16, 16, gop) == 0


def test_sps_differs_only_in_max_num_ref_frames():
    from gaussianavatars_b200 import video as V
    for w, h in [(48, 32), (550, 802), (1920, 1080)]:
        intra = V.parameter_sets(w, h, 20, Fraction(25))
        assert intra == O.parameter_sets(w, h, 20)
        for gop in (2, 25, 65535):
            sps, pps = V.parameter_sets(w, h, 20, Fraction(25), gop)
            assert (sps, pps) == S.parameter_sets(w, h, 20, 25, 1, gop)
            assert pps == intra[1]
            # the rbsp differs in one field: max_num_ref_frames ue(0) '1' -> ue(1) '010'
            a, b = (bin(int.from_bytes(r, "big"))[2:].zfill(8 * len(r)) for r in
                    (S._unescape(intra[0][1:]), S._unescape(sps[1:])))
            assert b[:29] == a[:29] and b[29:32] == "010" and b[32:].rstrip("0") == a[30:].rstrip("0")


def test_stream_parameter_sets_refuse_a_bad_gop(L):
    buf = (C.c_uint8 * 256)()
    assert L.gab200_h264_stream_parameter_sets(48, 32, 20, 25, 1, 0, buf, 256) == -1
    assert L.gab200_h264_stream_parameter_sets(48, 32, 20, 25, 1, 65536, buf, 256) == -1
    assert L.gab200_h264_stream_parameter_sets(48, 32, 20, 25, 1, 1, buf, 256) == \
        L.gab200_h264_parameter_sets(48, 32, 20, 25, 1, buf, 256)


def test_encode_stream_refusals(L):
    from gaussianavatars_b200 import _native as N
    w, h = 48, 32
    ok = dict(frames=1, qp=20, gop=25, rgb=256, state=256, scratch=256, out=256, stride=L.gab200_h264_p_bound(w, h),
              out_len=256)
    bad = [dict(gop=0), dict(gop=65536), dict(state=0), dict(state=264), dict(scratch=0), dict(scratch=128),
           dict(frames=0), dict(frames=65536), dict(qp=52), dict(qp=-1), dict(rgb=0), dict(out=0), dict(out_len=0),
           dict(stride=L.gab200_h264_p_bound(w, h) - 1)]
    n0 = N.launch_count()
    for change in bad:
        a = {**ok, **change}
        r = L.gab200_h264_encode_stream(a["frames"], h, w, a["qp"], a["gop"], a["rgb"], a["state"], a["scratch"],
                                        a["out"], a["stride"], a["out_len"], None)
        assert r == -1, change                  # GAB200_ERR_INVALID_ARGUMENT
    assert N.launch_count() == n0


@pytest.mark.parametrize("gop", [0, 65536, 2.0, True, "25"])
def test_video_writer_names_a_bad_gop(gop):
    import io

    from gaussianavatars_b200 import VideoWriter
    with pytest.raises(ValueError, match="gop"):
        VideoWriter(io.BytesIO(), 48, 32, gop=gop)


def _boxes(data, path):
    """The payload of the box at `path` (a list of four-character codes) in data, or None."""
    pos, end = 0, len(data)
    for kind in path:
        while pos < end:
            size = struct.unpack(">I", data[pos:pos + 4])[0]
            if size == 1:
                size = struct.unpack(">Q", data[pos + 8:pos + 16])[0]
            if data[pos + 4:pos + 8] == kind:
                break
            pos += size
        else:
            return None
        end = pos + size
        pos += 8
    return data[pos:end]


def test_moov_has_stss_exactly_when_gop_exceeds_one():
    from gaussianavatars_b200 import video as V
    sps, pps = V.parameter_sets(48, 32, 20, Fraction(25), 5)
    sizes = [100, 40, 41, 42, 43, 101, 44]
    plain = V.moov_box(sizes, 48, 48, 32, sps, pps, Fraction(25))
    assert _boxes(plain, [b"moov", b"trak", b"mdia", b"minf", b"stbl", b"stss"]) is None
    m = V.moov_box(sizes, 48, 48, 32, sps, pps, Fraction(25), [1, 6])
    assert _boxes(m, [b"moov", b"trak", b"mdia", b"minf", b"stbl", b"stss"]) == struct.pack(">IIII", 0, 2, 1, 6)
    assert m == S.moov(sizes, [True, False, False, False, False, True, False], 48, 48, 32, 20, 25, 1, 5)
