"""CPU: the deblocked H.264 stream surface without a launch -- gab200_h264_deblocked_scratch_bytes and the refusals
of gab200_h264_encode_deblocked, VideoWriter(deblock=), encode_video(deblock=) and export_trajectory(deblock=), and
parameter sets that are the same with and without the filter."""
import io
from fractions import Fraction

import pytest

from tests import h264_stream_oracle as S


@pytest.fixture(scope="module")
def L():
    from gaussianavatars_b200 import _native as N
    return N.lib()


def test_new_symbols_are_exported(L):
    from gaussianavatars_b200 import _native as N
    for name in ("gab200_h264_deblocked_scratch_bytes", "gab200_h264_encode_deblocked"):
        assert name in N.EXPORTED_SYMBOLS
        assert getattr(L, name) is not None


def test_deblocked_scratch_holds_the_plain_scratch_and_the_filtered_planes(L):
    for w, h in [(2, 2), (16, 16), (18, 34), (550, 802), (1920, 1080)]:
        nmb = ((w + 15) // 16) * ((h + 15) // 16)
        for k in (1, 3, 16):
            plain = L.gab200_h264_scratch_bytes(k, h, w)
            for gop in (1, 25):
                assert L.gab200_h264_deblocked_scratch_bytes(k, h, w, gop) == plain + k * ((384 * nmb + 255) // 256 * 256)
    for w, h in [(3, 2), (0, 16), (16, 8704 * 16)]:
        assert L.gab200_h264_deblocked_scratch_bytes(1, h, w, 1) == 0
    for gop in (0, 65536, -1):
        assert L.gab200_h264_deblocked_scratch_bytes(1, 16, 16, gop) == 0
    assert L.gab200_h264_deblocked_scratch_bytes(0, 16, 16, 1) == 0
    assert L.gab200_h264_deblocked_scratch_bytes(65536, 16, 16, 1) == 0


def test_encode_deblocked_refusals(L):
    from gaussianavatars_b200 import _native as N
    w, h = 48, 32
    ok = dict(frames=1, qp=20, gop=25, rgb=256, state=256, scratch=256, out=256, stride=L.gab200_h264_p_bound(w, h),
              out_len=256)
    bad = [dict(gop=0), dict(gop=65536), dict(state=0), dict(state=264), dict(scratch=0), dict(scratch=128),
           dict(frames=0), dict(frames=65536), dict(qp=52), dict(qp=-1), dict(rgb=0), dict(out=0), dict(out_len=0),
           dict(stride=L.gab200_h264_p_bound(w, h) - 1), dict(gop=1, stride=L.gab200_h264_bound(w, h) - 1),
           dict(gop=1, state=8)]
    n0 = N.launch_count()
    for change in bad:
        a = {**ok, **change}
        r = L.gab200_h264_encode_deblocked(a["frames"], h, a.get("w", w), a["qp"], a["gop"], a["rgb"], a["state"],
                                           a["scratch"], a["out"], a["stride"], a["out_len"], None)
        assert r == -1, change                  # GAB200_ERR_INVALID_ARGUMENT
    for width in (47, 0, 8704 * 16):
        r = L.gab200_h264_encode_deblocked(1, h, width, 20, 1, 256, None, 256, 256, 1 << 30, 256, None)
        assert r == -1, width
    assert N.launch_count() == n0


@pytest.mark.parametrize("deblock", [1, 0, None, "True", 1.0])
def test_a_deblock_that_is_not_a_bool_is_refused(deblock):
    from gaussianavatars_b200 import VideoWriter
    from gaussianavatars_b200.trajectory import export_trajectory
    with pytest.raises(ValueError, match="deblock"):
        VideoWriter(io.BytesIO(), 48, 32, gop=4, deblock=deblock)
    with pytest.raises(ValueError, match="deblock"):
        export_trajectory(None, None, "unused", bg=None, deblock=deblock)


def test_parameter_sets_do_not_depend_on_the_filter():
    # the PPS already sets deblocking_filter_control_present_flag: the slice header chooses, the SPS and PPS stay
    from gaussianavatars_b200 import video as V
    for w, h in [(48, 32), (550, 802), (1920, 1080)]:
        for gop in (1, 25):
            sps, pps = V.parameter_sets(w, h, 26, Fraction(25), gop)
            assert (sps, pps) == S.parameter_sets(w, h, 26, 25, 1, gop)
            rbsp = S._unescape(pps[1:])
            bits = bin(int.from_bytes(rbsp, "big"))[2:].zfill(8 * len(rbsp))
            # the PPS ends chroma_qp_index_offset se(0), deblocking_filter_control_present_flag 1,
            # constrained_intra_pred_flag 0, redundant_pic_cnt_present_flag 0 and the stop bit
            assert bits.rstrip("0").endswith("11001")
