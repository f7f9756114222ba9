"""CPU: the I_NxN H.264 stream surface without a launch -- gab200_h264_flags_scratch_bytes and the refusals of
gab200_h264_encode_flags, VideoWriter(intra4x4=), encode_video(intra4x4=) and export_trajectory(intra4x4=)."""
import io

import pytest

DEBLOCK, INTRA4X4 = 1, 2


@pytest.fixture(scope="module")
def L():
    from gaussianavatars_b200 import _native as N
    return N.lib()


def test_new_symbols_are_exported(L):
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import video as V
    for name in ("gab200_h264_flags_scratch_bytes", "gab200_h264_encode_flags"):
        assert name in N.EXPORTED_SYMBOLS
        assert getattr(L, name) is not None
    assert len(L.gab200_h264_encode_flags.argtypes) == 13
    assert (V.H264_DEBLOCK, V.H264_INTRA4X4) == (DEBLOCK, INTRA4X4)
    assert L.gab200_abi_version() == 3


def test_flags_scratch_is_the_existing_scratch_and_the_mode_array(L):
    for w, h in [(2, 2), (16, 16), (18, 34), (550, 802), (1920, 1080)]:
        nmb = ((w + 15) // 16) * ((h + 15) // 16)
        for k in (1, 3, 16):
            for gop in (1, 25):
                plain = L.gab200_h264_stream_scratch_bytes(k, h, w, gop)
                deblocked = L.gab200_h264_deblocked_scratch_bytes(k, h, w, gop)
                assert L.gab200_h264_flags_scratch_bytes(k, h, w, gop, 0) == plain
                assert L.gab200_h264_flags_scratch_bytes(k, h, w, gop, DEBLOCK) == deblocked
                modes = k * ((8 * nmb + 255) // 256 * 256)
                assert L.gab200_h264_flags_scratch_bytes(k, h, w, gop, INTRA4X4) == plain + modes
                assert L.gab200_h264_flags_scratch_bytes(k, h, w, gop, DEBLOCK | INTRA4X4) == deblocked + modes
    for w, h in [(3, 2), (0, 16), (16, 8704 * 16)]:
        assert L.gab200_h264_flags_scratch_bytes(1, h, w, 1, INTRA4X4) == 0
    for gop in (0, 65536, -1):
        assert L.gab200_h264_flags_scratch_bytes(1, 16, 16, gop, INTRA4X4) == 0
    for flags in (4, 8, 1 << 31, 0xFFFFFFFF):
        assert L.gab200_h264_flags_scratch_bytes(1, 16, 16, 1, flags) == 0
    assert L.gab200_h264_flags_scratch_bytes(0, 16, 16, 1, INTRA4X4) == 0
    assert L.gab200_h264_flags_scratch_bytes(65536, 16, 16, 1, INTRA4X4) == 0


def test_encode_flags_refusals(L):
    from gaussianavatars_b200 import _native as N
    w, h = 48, 32
    ok = dict(frames=1, qp=20, gop=25, flags=INTRA4X4, rgb=256, state=256, scratch=256, out=256,
              stride=L.gab200_h264_p_bound(w, h), out_len=256)
    bad = [dict(flags=4), dict(flags=INTRA4X4 | 16), dict(flags=0xFFFFFFFF), dict(gop=0), dict(gop=65536),
           dict(state=0), dict(state=264), dict(scratch=0), dict(scratch=128), dict(frames=0), dict(frames=65536),
           dict(qp=52), dict(qp=-1), dict(rgb=0), dict(out=0), dict(out_len=0),
           dict(stride=L.gab200_h264_p_bound(w, h) - 1), dict(gop=1, stride=L.gab200_h264_bound(w, h) - 1),
           dict(gop=1, state=8), dict(flags=DEBLOCK | INTRA4X4, state=0)]
    n0 = N.launch_count()
    for change in bad:
        a = {**ok, **change}
        r = L.gab200_h264_encode_flags(a["frames"], h, w, a["qp"], a["gop"], a["flags"], a["rgb"], a["state"],
                                       a["scratch"], a["out"], a["stride"], a["out_len"], None)
        assert r == -1, change                  # GAB200_ERR_INVALID_ARGUMENT
    for width in (47, 0, 8704 * 16):
        r = L.gab200_h264_encode_flags(1, h, width, 20, 1, INTRA4X4, 256, None, 256, 256, 1 << 30, 256, None)
        assert r == -1, width
    assert N.launch_count() == n0


@pytest.mark.parametrize("intra4x4", [1, 0, None, "True", 1.0])
def test_an_intra4x4_that_is_not_a_bool_is_refused(intra4x4):
    from gaussianavatars_b200 import VideoWriter, encode_video
    from gaussianavatars_b200.trajectory import export_trajectory
    with pytest.raises(ValueError, match="intra4x4"):
        VideoWriter(io.BytesIO(), 48, 32, gop=4, intra4x4=intra4x4)
    with pytest.raises(ValueError, match="intra4x4"):
        VideoWriter(io.BytesIO(), 48, 32, deblock=True, intra4x4=intra4x4)
    with pytest.raises(ValueError, match="intra4x4"):
        export_trajectory(None, None, "unused", bg=None, intra4x4=intra4x4)
    with pytest.raises(ValueError, match="intra4x4"):
        encode_video(None, intra4x4=intra4x4)
