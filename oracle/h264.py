"""A plain restatement of the device H.264 encoder (csrc/h264.cu) and of the MP4 muxer (gaussianavatars_b200/video.py),
written from ITU-T H.264 (clauses 7, 8.3, 8.5, 9.2 and Annex A) -- what tests/test_gpu_video.py compares the device's
bytes with, and what FFmpeg's decoder referees in tests/test_oracle_h264.py.

    out = encode_frame(rgb, qp)        # (H,W,3) uint8 -> dict(sample=AVCC bytes, recon=(Y, Cb, Cr), report=set, ...)
    sps, pps = parameter_sets(W, H, qp, fps_num, fps_den)
    data = mp4([out["sample"], ...], W, H, qp, fps_num, fps_den)

The stream: Constrained Baseline, every picture one IDR slice, CAVLC, deblocking off, a fixed QP.  Each macroblock is
I_16x16 with the luma and chroma modes of least SATD (ties: the lowest mode number), or I_PCM when a level falls
outside +-2063 or its CAVLC bits exceed I_PCM's 9 + 3072.  With deblocking off, every conforming decoder outputs exactly
`recon`.  Every sample carries idr_pic_id 1; mp4() sets idr_pic_id 2 on the odd-numbered samples (ue(1) and ue(2) have
the same length, so it is one bit of byte 6 of the sample).

The macroblocks of an anti-diagonal (mbx + mby = d) read only reconstructed samples of earlier diagonals, so each
diagonal's prediction, transforms and reconstruction are done for all its macroblocks at once in numpy; the CAVLC
of each macroblock is written by a small Python bit writer.
"""
from __future__ import annotations

import struct
from fractions import Fraction

import numpy as np

MAX_LEVEL = 2063            # |level| that level_prefix <= 15 codes at every suffixLength
PCM_BITS = 9 + 384 * 8      # ue(25) + the samples, before pcm_alignment_zero_bits
HEADER_BITS = 22            # the slice header after the NAL header byte (see slice_header)
ZIGZAG = np.array([0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15])
CHROMA_QP = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
MF = np.array([[13107, 5243, 8066], [11916, 4660, 7490], [10082, 4194, 6554], [9362, 3647, 5825], [8192, 3355, 5243],
               [7282, 2893, 4559]], np.int64)     # forward quantisation multipliers
V = np.array([[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]], np.int64)  # normAdjust4x4 (8.5.9)
POS = np.array([[0 if (i % 2 == 0 and j % 2 == 0) else 1 if (i % 2 and j % 2) else 2 for j in range(4)] for i in range(4)])
CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
HD = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
H2 = np.array([[1, 1], [1, -1]], np.int64)

# Table A-1: (level_idc, MaxMBPS, MaxFS); level 1b is not used
LEVELS = [(10, 1485, 99), (11, 3000, 396), (12, 6000, 396), (13, 11880, 396), (20, 11880, 396), (21, 19800, 792),
          (22, 20250, 1620), (30, 40500, 1620), (31, 108000, 3600), (32, 216000, 5120), (40, 245760, 8192),
          (41, 245760, 8192), (42, 522240, 8704), (50, 589824, 22080), (51, 983040, 36864), (52, 2073600, 36864)]

# Table 9-5, [TrailingOnes + 4 TotalCoeff]: code lengths and values for 0 <= nC < 2, 2 <= nC < 4, 4 <= nC < 8, 8 <= nC
COEFF_TOKEN_LEN = [
    [1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9,
     13, 13, 13, 10, 14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15,
     16, 16, 16, 16, 16, 16, 16, 16],
    [2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6, 11, 11, 11, 7,
     12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13,
     14, 14, 14, 14],
    [4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4, 8, 7, 7, 5,
     8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10],
    [6, 0, 0, 0, 6, 6, 0, 0, 6, 6, 6, 0] + [6] * 56,
]
COEFF_TOKEN_CODE = [
    [1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4, 8, 10, 13, 4,
     15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12,
     4, 6, 5, 8],
    [3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4, 11, 14, 13, 4,
     15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8, 9, 8, 10, 1,
     7, 6, 5, 4],
    [15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9, 8, 10, 9, 8,
     15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12, 9, 12, 11, 10,
     5, 8, 7, 6, 1, 4, 3, 2],
    [3, 0, 0, 0, 0, 1, 0, 0, 4, 5, 6, 0] + list(range(8, 64)),
]
CHROMA_DC_TOKEN_LEN = [2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7]      # nC = -1
CHROMA_DC_TOKEN_CODE = [1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0]
# Tables 9-7 and 9-8, [TotalCoeff - 1][total_zeros]
TOTAL_ZEROS_LEN = [
    [1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9], [3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6],
    [4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6], [5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5],
    [4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5], [6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6], [6, 5, 3, 3, 3, 2, 3, 4, 3, 6],
    [6, 4, 5, 3, 2, 2, 3, 3, 6], [6, 6, 4, 2, 2, 3, 2, 5], [5, 5, 3, 2, 2, 2, 4], [4, 4, 3, 3, 1, 3], [4, 4, 2, 1, 3],
    [3, 3, 1, 2], [2, 2, 1], [1, 1]]
TOTAL_ZEROS_CODE = [
    [1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1], [7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0],
    [5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0], [3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0],
    [5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 5, 4, 3, 3, 2, 1, 1, 0],
    [1, 1, 1, 3, 3, 2, 2, 1, 0], [1, 0, 1, 3, 2, 1, 1, 1], [1, 0, 1, 3, 2, 1, 1], [0, 1, 1, 2, 1, 3], [0, 1, 1, 1, 1],
    [0, 1, 1, 1], [0, 1, 1], [0, 1]]
CHROMA_DC_TOTAL_ZEROS_LEN = [[1, 2, 3, 3], [1, 2, 2], [1, 1]]
CHROMA_DC_TOTAL_ZEROS_CODE = [[1, 1, 1, 0], [1, 1, 0], [1, 0]]
# Table 9-10, [min(zerosLeft, 7) - 1][run_before]
RUN_BEFORE_LEN = [[1, 1], [1, 2, 2], [2, 2, 2, 2], [2, 2, 2, 3, 3], [2, 2, 3, 3, 3, 3], [2, 3, 3, 3, 3, 3, 3],
                  [3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
RUN_BEFORE_CODE = [[1, 0], [1, 1, 0], [3, 2, 1, 0], [3, 2, 1, 1, 0], [3, 2, 3, 2, 1, 0], [3, 0, 1, 3, 2, 5, 4],
                   [7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1]]
TOKEN_TABLE_NAMES = ("nC0-1", "nC2-3", "nC4-7", "nC8+", "chromaDC")


# ---- sizes, levels, bound ----------------------------------------------------------------------------------------
def coded_size(width: int, height: int) -> tuple:
    return (width + 15) // 16 * 16, (height + 15) // 16 * 16


def level_idc(width: int, height: int, fps: float = 25.0):
    """The smallest level of Table A-1 whose MaxFS, sqrt(8 MaxFS) side limit and MaxMBPS cover the size at `fps`
    (level 5.2 when only the rate exceeds every level); None when the frame exceeds level 5.2's MaxFS or side."""
    wm, hm = (width + 15) // 16, (height + 15) // 16
    fs = wm * hm
    for idc, mbps, maxfs in LEVELS:
        if fs <= maxfs and wm * wm <= 8 * maxfs and hm * hm <= 8 * maxfs and fs * fps <= mbps:
            return idc
    if fs <= 36864 and wm * wm <= 8 * 36864 and hm * hm <= 8 * 36864:
        return 52
    return None


def bound(width: int, height: int) -> int:
    """The largest sample of a width x height frame: 4 + 1 + n + ceil(n / 2) bytes for the n bytes of a slice whose
    every macroblock is an I_PCM one at its worst alignment (emulation prevention adds at most one byte per two); -1
    for an odd or empty size or one above level 5.2."""
    if width <= 0 or height <= 0 or width % 2 or height % 2 or level_idc(width, height, 0) is None:
        return -1
    nmb = ((width + 15) // 16) * ((height + 15) // 16)
    n = (HEADER_BITS + nmb * (PCM_BITS + 7) + 1 + 7) // 8
    return 5 + n + (n + 1) // 2


# ---- bit writing -------------------------------------------------------------------------------------------------
class Bits:
    def __init__(self):
        self.parts = []
        self.n = 0

    def u(self, value: int, length: int):
        if length:
            self.parts.append(format(value, "0%db" % length))
            self.n += length

    def ue(self, v: int):
        x = v + 1
        L = x.bit_length()
        self.u(x, 2 * L - 1)

    def se(self, v: int):
        self.ue(2 * v - 1 if v > 0 else -2 * v)

    def bits(self) -> str:
        return "".join(self.parts)


def to_bytes(bits: str) -> bytes:
    bits = bits + "0" * (-len(bits) % 8)
    return int(bits, 2).to_bytes(len(bits) // 8, "big") if bits else b""


def emulation_prevention(rbsp: bytes) -> tuple:
    """(escaped bytes, number of 0x03 bytes inserted): 0x03 before any byte <= 3 that follows two zero bytes."""
    out = bytearray()
    zeros = inserted = 0
    for b in rbsp:
        if zeros >= 2 and b <= 3:
            out.append(3)
            zeros = 0
            inserted += 1
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out), inserted


def nal(nal_type: int, rbsp: bytes) -> bytes:
    return bytes([0x60 | nal_type]) + emulation_prevention(rbsp)[0]


def rbsp_trailing(b: Bits) -> str:
    b.u(1, 1)
    return b.bits() + "0" * (-b.n % 8)


def parameter_sets(width: int, height: int, qp: int, fps_num: int = 25, fps_den: int = 1) -> tuple:
    """(SPS, PPS) NAL units, each with its header byte."""
    wc, hc = coded_size(width, height)
    b = Bits()
    b.u(66, 8)                      # profile_idc: Baseline
    b.u(0xC0, 8)                    # constraint_set0_flag = constraint_set1_flag = 1: Constrained Baseline
    b.u(level_idc(width, height, Fraction(fps_num, fps_den)), 8)
    b.ue(0)                         # seq_parameter_set_id
    b.ue(0)                         # log2_max_frame_num_minus4
    b.ue(2)                         # pic_order_cnt_type
    b.ue(0)                         # max_num_ref_frames
    b.u(0, 1)                       # gaps_in_frame_num_value_allowed_flag
    b.ue(wc // 16 - 1)
    b.ue(hc // 16 - 1)
    b.u(1, 1)                       # frame_mbs_only_flag
    b.u(1, 1)                       # direct_8x8_inference_flag
    crop = wc != width or hc != height
    b.u(int(crop), 1)
    if crop:
        b.ue(0)
        b.ue((wc - width) // 2)
        b.ue(0)
        b.ue((hc - height) // 2)
    b.u(1, 1)                       # vui_parameters_present_flag
    b.u(0, 1)                       # aspect_ratio_info_present_flag
    b.u(0, 1)                       # overscan_info_present_flag
    b.u(1, 1)                       # video_signal_type_present_flag
    b.u(5, 3)                       # video_format: unspecified
    b.u(0, 1)                       # video_full_range_flag: limited range
    b.u(1, 1)                       # colour_description_present_flag
    b.u(2, 8)                       # colour_primaries: unspecified
    b.u(2, 8)                       # transfer_characteristics: unspecified
    b.u(6, 8)                       # matrix_coefficients: BT.601 (SMPTE 170M)
    b.u(0, 1)                       # chroma_loc_info_present_flag
    b.u(1, 1)                       # timing_info_present_flag
    b.u(fps_den, 32)                # num_units_in_tick
    b.u(2 * fps_num, 32)            # time_scale (two ticks per frame)
    b.u(1, 1)                       # fixed_frame_rate_flag
    b.u(0, 1)                       # nal_hrd_parameters_present_flag
    b.u(0, 1)                       # vcl_hrd_parameters_present_flag
    b.u(0, 1)                       # pic_struct_present_flag
    b.u(0, 1)                       # bitstream_restriction_flag
    sps = nal(7, to_bytes(rbsp_trailing(b)))
    b = Bits()
    b.ue(0)                         # pic_parameter_set_id
    b.ue(0)                         # seq_parameter_set_id
    b.u(0, 1)                       # entropy_coding_mode_flag: CAVLC
    b.u(0, 1)                       # bottom_field_pic_order_in_frame_present_flag
    b.ue(0)                         # num_slice_groups_minus1
    b.ue(0)
    b.ue(0)                         # num_ref_idx_l0/l1_default_active_minus1
    b.u(0, 1)                       # weighted_pred_flag
    b.u(0, 2)                       # weighted_bipred_idc
    b.se(qp - 26)                   # pic_init_qp_minus26
    b.se(0)                         # pic_init_qs_minus26
    b.se(0)                         # chroma_qp_index_offset
    b.u(1, 1)                       # deblocking_filter_control_present_flag
    b.u(0, 1)                       # constrained_intra_pred_flag
    b.u(0, 1)                       # redundant_pic_cnt_present_flag
    pps = nal(8, to_bytes(rbsp_trailing(b)))
    return sps, pps


def slice_header(b: Bits, idr_pic_id: int = 1):
    b.ue(0)                         # first_mb_in_slice
    b.ue(7)                         # slice_type: I (all slices of the picture)
    b.ue(0)                         # pic_parameter_set_id
    b.u(0, 4)                       # frame_num
    b.ue(idr_pic_id)
    b.u(0, 1)                       # no_output_of_prior_pics_flag
    b.u(0, 1)                       # long_term_reference_flag
    b.se(0)                         # slice_qp_delta
    b.ue(1)                         # disable_deblocking_filter_idc


# ---- colour conversion -------------------------------------------------------------------------------------------
def rgb_to_yuv(rgb: np.ndarray) -> tuple:
    """BT.601 limited range in integers; chroma from the sum of each 2x2 block; planes padded to whole macroblocks by
    edge replication.  Y = ((66 R + 129 G + 25 B + 128) >> 8) + 16; with R4, G4, B4 the 2x2 sums,
    Cb = ((-38 R4 - 74 G4 + 112 B4 + 512) >> 10) + 128, Cr = ((112 R4 - 94 G4 - 18 B4 + 512) >> 10) + 128."""
    H, W, _ = rgb.shape
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16

    def s4(p):
        return p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]

    r4, g4, b4 = s4(r), s4(g), s4(b)
    cb = ((-38 * r4 - 74 * g4 + 112 * b4 + 512) >> 10) + 128
    cr = ((112 * r4 - 94 * g4 - 18 * b4 + 512) >> 10) + 128
    wc, hc = coded_size(W, H)
    pad = lambda p, f: np.pad(p, ((0, (hc - H) // f), (0, (wc - W) // f)), mode="edge")   # noqa: E731
    return pad(y, 1), pad(cb, 2), pad(cr, 2)


# ---- prediction (8.3.3, 8.3.4), vectorised over the macroblocks of a diagonal ------------------------------------
def predict(top, left, tl, has_top, has_left, n: int, chroma: bool) -> np.ndarray:
    """(M, 4, n, n) predictions of the four modes (luma order V, H, DC, Plane; chroma order DC, H, V, Plane) from
    top (M, n), left (M, n), tl (M,); unavailable modes are filled but never chosen."""
    M = top.shape[0]
    vert = np.broadcast_to(top[:, None, :], (M, n, n))
    horz = np.broadcast_to(left[:, :, None], (M, n, n))
    if not chroma:
        st, sl = top.sum(1), left.sum(1)
        dc = np.where(has_top & has_left, (st + sl + 16) >> 5,
                      np.where(has_top, (st + 8) >> 4, np.where(has_left, (sl + 8) >> 4, 128)))
        dcp = np.broadcast_to(dc[:, None, None], (M, n, n))
        xs = np.arange(8)
        topx = np.concatenate([tl[:, None], top], 1)        # index k + 1 holds p[k, -1]
        leftx = np.concatenate([tl[:, None], left], 1)
        Hh = ((xs + 1) * (topx[:, 9 + xs] - topx[:, 7 - xs])).sum(1)
        Vv = ((xs + 1) * (leftx[:, 9 + xs] - leftx[:, 7 - xs])).sum(1)
        a = 16 * (left[:, 15] + top[:, 15])
        bb, cc = (5 * Hh + 32) >> 6, (5 * Vv + 32) >> 6
        ctr = 7
    else:
        dcp = np.empty((M, n, n), np.int64)
        for by in range(2):
            for bx in range(2):
                st, sl = top[:, 4 * bx:4 * bx + 4].sum(1), left[:, 4 * by:4 * by + 4].sum(1)
                both = np.where(has_top & has_left, (st + sl + 4) >> 3,
                                np.where(has_top, (st + 2) >> 2, np.where(has_left, (sl + 2) >> 2, 128)))
                if bx == by:
                    v = both
                elif bx == 1:       # top-right block: top first
                    v = np.where(has_top, (st + 2) >> 2, np.where(has_left, (sl + 2) >> 2, 128))
                else:               # bottom-left block: left first
                    v = np.where(has_left, (sl + 2) >> 2, np.where(has_top, (st + 2) >> 2, 128))
                dcp[:, 4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = v[:, None, None]
        xs = np.arange(4)
        topx = np.concatenate([tl[:, None], top], 1)
        leftx = np.concatenate([tl[:, None], left], 1)
        Hh = ((xs + 1) * (topx[:, 5 + xs] - topx[:, 3 - xs])).sum(1)
        Vv = ((xs + 1) * (leftx[:, 5 + xs] - leftx[:, 3 - xs])).sum(1)
        a = 16 * (left[:, 7] + top[:, 7])
        bb, cc = (34 * Hh + 32) >> 6, (34 * Vv + 32) >> 6
        ctr = 3
    g = np.arange(n) - ctr
    plane = np.clip((a[:, None, None] + bb[:, None, None] * g[None, None, :] + cc[:, None, None] * g[None, :, None]
                     + 16) >> 5, 0, 255)
    modes = [vert, horz, dcp, plane] if not chroma else [dcp, horz, vert, plane]
    return np.stack(modes, 1).astype(np.int64)


def blocks(x: np.ndarray) -> np.ndarray:
    """(..., 4a, 4b) -> (..., a, b, 4, 4): the 4x4 blocks, [block row, block column, y, x]."""
    *lead, h, w = x.shape
    return x.reshape(*lead, h // 4, 4, w // 4, 4).swapaxes(-3, -2)


def unblocks(x: np.ndarray) -> np.ndarray:
    *lead, a, b, _, _ = x.shape
    return x.swapaxes(-3, -2).reshape(*lead, 4 * a, 4 * b)


def satd(res: np.ndarray) -> np.ndarray:
    """Sum over the 4x4 blocks of |HD r HD| -- res (..., h, w) -> (...)."""
    t = HD @ blocks(res) @ HD
    return np.abs(t).sum(axis=(-4, -3, -2, -1))


def choose(pred, src, avail) -> np.ndarray:
    """Index of the available mode of least SATD (pred (M, 4, ...), src (M, ...) or a list of planes); first on ties."""
    cost = sum(satd(s[:, None] - p) for p, s in zip(pred, src))
    cost = np.where(avail, cost, np.iinfo(np.int64).max)
    return np.argmin(cost, 1)


# ---- transform, quantisation, reconstruction (8.5) ---------------------------------------------------------------
def quant(c, qp, mf, dc):
    qbits = 15 + qp // 6
    f = (1 << qbits) // 3
    if dc:
        q = (np.abs(c) * mf + 2 * f) >> (qbits + 1)
    else:
        q = (np.abs(c) * mf + f) >> qbits
    return np.sign(c) * q


def dequant_ac(c, qp):
    ls = 16 * V[qp % 6][POS]
    if qp >= 24:
        return (c * ls) << (qp // 6 - 4)
    return (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)


def idct4(d):
    """8.5.12.2: rows (horizontal) first, then columns; (..., 4, 4) -> residual (h + 32) >> 6."""
    e0, e1 = d[..., 0] + d[..., 2], d[..., 0] - d[..., 2]
    e2, e3 = (d[..., 1] >> 1) - d[..., 3], d[..., 1] + (d[..., 3] >> 1)
    f = np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)
    g0, g1 = f[..., 0, :] + f[..., 2, :], f[..., 0, :] - f[..., 2, :]
    g2, g3 = (f[..., 1, :] >> 1) - f[..., 3, :], f[..., 1, :] + (f[..., 3, :] >> 1)
    h = np.stack([g0 + g3, g1 + g2, g1 - g2, g0 - g3], -2)
    return (h + 32) >> 6


def code_luma(res, qp):
    """res (M, 16, 16) -> (dc levels (M, 4, 4) [block row, block column], ac levels (M, 4, 4, 4, 4) with 0 at [.., 0,
    0], reconstructed residual (M, 16, 16))."""
    w = CF @ blocks(res) @ CF.T
    t = (HD @ w[..., 0, 0] @ HD) >> 1
    dcl = quant(t, qp, MF[qp % 6, 0], True)
    acl = quant(w, qp, MF[qp % 6][POS], False)
    acl[..., 0, 0] = 0
    return dcl, acl, recon_luma(dcl, acl, qp)


def recon_luma(dcl, acl, qp):
    """8.5.10 and 8.5.12: the residual (M, 16, 16) of Intra16x16 DC levels (M, 4, 4) and AC levels (M, 4, 4, 4, 4)."""
    f = HD @ dcl @ HD
    ls = 16 * V[qp % 6, 0]
    dcy = (f * ls) << (qp // 6 - 6) if qp >= 36 else (f * ls + (1 << (5 - qp // 6))) >> (6 - qp // 6)
    d = dequant_ac(acl, qp)
    d[..., 0, 0] = dcy
    return unblocks(idct4(d))


def code_chroma(res, qpc):
    """res (M, 8, 8) -> (dc levels (M, 2, 2), ac levels (M, 2, 2, 4, 4), reconstructed residual (M, 8, 8))."""
    w = CF @ blocks(res) @ CF.T
    t = H2 @ w[..., 0, 0] @ H2
    dcl = quant(t, qpc, MF[qpc % 6, 0], True)
    acl = quant(w, qpc, MF[qpc % 6][POS], False)
    acl[..., 0, 0] = 0
    return dcl, acl, recon_chroma(dcl, acl, qpc)


def recon_chroma(dcl, acl, qpc):
    """8.5.11 and 8.5.12: the residual (M, 8, 8) of chroma DC levels (M, 2, 2) and AC levels (M, 2, 2, 4, 4)."""
    f = H2 @ dcl @ H2
    dcc = ((f * (16 * V[qpc % 6, 0])) << (qpc // 6)) >> 5
    d = dequant_ac(acl, qpc)
    d[..., 0, 0] = dcc
    return unblocks(idct4(d))


# ---- CAVLC (9.2) -------------------------------------------------------------------------------------------------
def residual_block(b: Bits, coeffs, nc: int, report: set):
    """Writes one residual_block_cavlc of the coefficient list `coeffs` (scan order) with context nC (-1: chroma DC);
    returns TotalCoeff."""
    coeffs = [int(v) for v in coeffs]
    maxn = len(coeffs)
    nz = [i for i, v in enumerate(coeffs) if v]
    total = len(nz)
    levels = [coeffs[i] for i in reversed(nz)]           # highest frequency first
    t1 = 0
    for v in levels:
        if abs(v) == 1 and t1 < 3:
            t1 += 1
        else:
            break
    if nc < 0:
        b.u(CHROMA_DC_TOKEN_CODE[4 * total + t1], CHROMA_DC_TOKEN_LEN[4 * total + t1])
        report.add(("coeff_token", "chromaDC"))
    else:
        tab = 0 if nc < 2 else 1 if nc < 4 else 2 if nc < 8 else 3
        b.u(COEFF_TOKEN_CODE[tab][4 * total + t1], COEFF_TOKEN_LEN[tab][4 * total + t1])
        report.add(("coeff_token", TOKEN_TABLE_NAMES[tab]))
    if total == 0:
        return 0
    for v in levels[:t1]:
        b.u(int(v < 0), 1)
    sl = 1 if total > 10 and t1 < 3 else 0
    for i, v in enumerate(levels[t1:]):
        code = 2 * v - 2 if v > 0 else -2 * v - 1
        if i == 0 and t1 < 3:
            code -= 2
        report.add(("suffixLength", sl))
        if sl == 0:
            if code < 14:
                prefix, suffix, slen = code, 0, 0
            elif code < 30:
                prefix, suffix, slen = 14, code - 14, 4
            else:
                prefix, suffix, slen = 15, code - 30, 12
        elif code < (15 << sl):
            prefix, suffix, slen = code >> sl, code & ((1 << sl) - 1), sl
        else:
            prefix, suffix, slen = 15, code - (15 << sl), 12
        assert suffix < (1 << slen) or slen == 0 and suffix == 0, "level out of Baseline's range"
        report.add(("level_prefix", prefix))
        b.u(1, prefix + 1)
        b.u(suffix, slen)
        if sl == 0:
            sl = 1
        if abs(v) > (3 << (sl - 1)) and sl < 6:
            sl += 1
    zeros = nz[-1] + 1 - total
    if total < maxn:
        if nc < 0:
            b.u(CHROMA_DC_TOTAL_ZEROS_CODE[total - 1][zeros], CHROMA_DC_TOTAL_ZEROS_LEN[total - 1][zeros])
            report.add(("total_zeros", "chromaDC", total))
        else:
            b.u(TOTAL_ZEROS_CODE[total - 1][zeros], TOTAL_ZEROS_LEN[total - 1][zeros])
            report.add(("total_zeros", "luma", total))
    left = zeros
    for k in range(total - 1, 0, -1):                    # every coefficient but the lowest-frequency one
        if left <= 0:
            break
        run = nz[k] - nz[k - 1] - 1
        t = min(left, 7) - 1
        b.u(RUN_BEFORE_CODE[t][run], RUN_BEFORE_LEN[t][run])
        report.add(("run_before", min(left, 7)))
        left -= run
    return total


def nc_of(tot: np.ndarray, x: int, y: int) -> int:
    """nC of the 4x4 block at (x, y) of a totals grid: the rounded mean of the available left and top totals."""
    a = int(tot[y, x - 1]) if x > 0 else None
    bt = int(tot[y - 1, x]) if y > 0 else None
    if a is not None and bt is not None:
        return (a + bt + 1) >> 1
    return a if a is not None else bt if bt is not None else 0


LUMA_BLK = [((i8 % 2) * 2 + i4 % 2, (i8 // 2) * 2 + i4 // 2) for i8 in range(4) for i4 in range(4)]  # (bx, by)


def macroblock_bits(mx, my, lmode, cmode, dcl, acl, cdcl, cacl, tl_, tc_, report):
    """The I_16x16 macroblock_layer's bits; fills its totals into the grids tl_ (luma) and tc_ (Cb, Cr)."""
    cbpl = 15 if np.any(acl) else 0
    cbpc = 2 if np.any(cacl) else 1 if np.any(cdcl) else 0
    for k, (bx, by) in enumerate(LUMA_BLK):
        tl_[4 * my + by, 4 * mx + bx] = np.count_nonzero(acl[by, bx]) if cbpl else 0
    for c in range(2):
        for by in range(2):
            for bx in range(2):
                tc_[c][2 * my + by, 2 * mx + bx] = np.count_nonzero(cacl[c, by, bx]) if cbpc == 2 else 0
    b = Bits()
    b.ue(1 + lmode + 4 * cbpc + (12 if cbpl else 0))
    b.ue(cmode)
    b.se(0)                                              # mb_qp_delta
    residual_block(b, dcl.reshape(16)[ZIGZAG], nc_of(tl_, 4 * mx, 4 * my), report)
    if cbpl:
        for bx, by in LUMA_BLK:
            residual_block(b, acl[by, bx].reshape(16)[ZIGZAG[1:]], nc_of(tl_, 4 * mx + bx, 4 * my + by), report)
    if cbpc:
        for c in range(2):
            residual_block(b, cdcl[c].reshape(4), -1, report)
    if cbpc == 2:
        for c in range(2):
            for by in range(2):
                for bx in range(2):
                    residual_block(b, cacl[c, by, bx].reshape(16)[ZIGZAG[1:]],
                                   nc_of(tc_[c], 2 * mx + bx, 2 * my + by), report)
    return b


# ---- the encode --------------------------------------------------------------------------------------------------
def encode_frame(rgb: np.ndarray, qp: int) -> dict:
    """One frame -> dict(sample: the AVCC sample (4-byte length + IDR slice NAL, idr_pic_id 1), recon: (Y, Cb, Cr)
    cropped to the frame, modes: (luma (Hm, Wm), chroma (Hm, Wm), pcm (Hm, Wm)), report: the CAVLC paths reached)."""
    rgb = np.asarray(rgb, np.uint8)
    H, W, _ = rgb.shape
    if bound(W, H) < 0:
        raise ValueError(f"no H.264 frame of {W}x{H}")
    if not 0 <= qp <= 51:
        raise ValueError(f"qp must be in 0..51, got {qp}")
    qpc = CHROMA_QP[qp]
    ys, cbs, crs = rgb_to_yuv(rgb)
    hc, wc = ys.shape
    hm, wm = hc // 16, wc // 16
    ry, rcb, rcr = np.zeros_like(ys), np.zeros_like(cbs), np.zeros_like(crs)
    tl_ = np.zeros((4 * hm, 4 * wm), np.int64)
    tc_ = [np.zeros((2 * hm, 2 * wm), np.int64) for _ in range(2)]
    lmodes, cmodes = np.zeros((hm, wm), np.int64), np.zeros((hm, wm), np.int64)
    pcm = np.zeros((hm, wm), bool)
    mbbits = {}
    report = set()
    for d in range(wm + hm - 1):
        mx = np.arange(max(0, d - hm + 1), min(d, wm - 1) + 1)
        my = d - mx
        has_l, has_t = mx > 0, my > 0
        M = len(mx)
        yy = (16 * my)[:, None] + np.arange(16)
        xx = (16 * mx)[:, None] + np.arange(16)
        src = ys[yy[:, :, None], xx[:, None, :]]
        top = np.where(has_t[:, None], ry[np.maximum(16 * my - 1, 0)[:, None], xx], 0)
        left = np.where(has_l[:, None], ry[yy, np.maximum(16 * mx - 1, 0)[:, None]], 0)
        tlv = np.where(has_t & has_l, ry[np.maximum(16 * my - 1, 0), np.maximum(16 * mx - 1, 0)], 0)
        pl = predict(top, left, tlv, has_t, has_l, 16, False)
        lav = np.stack([has_t, has_l, np.ones(M, bool), has_t & has_l], 1)
        lm = choose([pl], [src], lav)
        pred = pl[np.arange(M), lm]
        dcl, acl, rres = code_luma(src - pred, qp)
        rec = np.clip(pred + rres, 0, 255)
        cy = (8 * my)[:, None] + np.arange(8)
        cx = (8 * mx)[:, None] + np.arange(8)
        csrc, cpred_all = [], []
        for plane, rp in ((cbs, rcb), (crs, rcr)):
            csrc.append(plane[cy[:, :, None], cx[:, None, :]])
            top = np.where(has_t[:, None], rp[np.maximum(8 * my - 1, 0)[:, None], cx], 0)
            left = np.where(has_l[:, None], rp[cy, np.maximum(8 * mx - 1, 0)[:, None]], 0)
            tlv = np.where(has_t & has_l, rp[np.maximum(8 * my - 1, 0), np.maximum(8 * mx - 1, 0)], 0)
            cpred_all.append(predict(top, left, tlv, has_t, has_l, 8, True))
        cav = np.stack([np.ones(M, bool), has_l, has_t, has_t & has_l], 1)
        cm = choose(cpred_all, csrc, cav)
        cres = [code_chroma(s - p[np.arange(M), cm], qpc) for s, p in zip(csrc, cpred_all)]
        crec = [np.clip(p[np.arange(M), cm] + r[2], 0, 255) for p, r in zip(cpred_all, cres)]
        cdcl = np.stack([r[0] for r in cres], 1)          # (M, 2, 2, 2)
        cacl = np.stack([r[1] for r in cres], 1)          # (M, 2, 2, 2, 4, 4)
        for i in range(M):
            x, y = int(mx[i]), int(my[i])
            over = max(np.abs(dcl[i]).max(), np.abs(acl[i]).max(), np.abs(cdcl[i]).max(), np.abs(cacl[i]).max())
            b = None
            if over <= MAX_LEVEL:
                rep = set()
                b = macroblock_bits(x, y, int(lm[i]), int(cm[i]), dcl[i], acl[i], cdcl[i], cacl[i], tl_, tc_, rep)
                if b.n > PCM_BITS:
                    b = None
                else:
                    report |= rep
            if b is None:
                pcm[y, x] = True
                tl_[4 * y:4 * y + 4, 4 * x:4 * x + 4] = 16
                for t in tc_:
                    t[2 * y:2 * y + 2, 2 * x:2 * x + 2] = 16
                ry[16 * y:16 * y + 16, 16 * x:16 * x + 16] = src[i]
                rcb[8 * y:8 * y + 8, 8 * x:8 * x + 8] = csrc[0][i]
                rcr[8 * y:8 * y + 8, 8 * x:8 * x + 8] = csrc[1][i]
                report.add(("mb", "I_PCM"))
            else:
                mbbits[(y, x)] = b.bits()
                lmodes[y, x], cmodes[y, x] = lm[i], cm[i]
                ry[16 * y:16 * y + 16, 16 * x:16 * x + 16] = rec[i]
                rcb[8 * y:8 * y + 8, 8 * x:8 * x + 8] = crec[0][i]
                rcr[8 * y:8 * y + 8, 8 * x:8 * x + 8] = crec[1][i]
                report.add(("luma_mode", int(lm[i])))
                report.add(("chroma_mode", int(cm[i])))
    b = Bits()
    slice_header(b)
    assert b.n == HEADER_BITS
    parts = [b.bits()]
    n = b.n
    for y in range(hm):
        for x in range(wm):
            if pcm[y, x]:
                head = "000011010" + "0" * (-(n + 9) % 8)            # ue(25), pcm_alignment_zero_bits
                samples = np.concatenate([ys[16 * y:16 * y + 16, 16 * x:16 * x + 16].ravel(),
                                          cbs[8 * y:8 * y + 8, 8 * x:8 * x + 8].ravel(),
                                          crs[8 * y:8 * y + 8, 8 * x:8 * x + 8].ravel()])
                s = head + "".join(format(int(v), "08b") for v in samples)
            else:
                s = mbbits[(y, x)]
            parts.append(s)
            n += len(s)
    parts.append("1")                                                  # rbsp_stop_one_bit
    rbsp = to_bytes("".join(parts))
    esc, inserted = emulation_prevention(rbsp)
    if inserted:
        report.add(("emulation_prevention",))
    body = b"\x65" + esc
    sample = struct.pack(">I", len(body)) + body
    assert len(sample) <= bound(W, H)
    recon = (ry[:H, :W].astype(np.uint8), rcb[:H // 2, :W // 2].astype(np.uint8), rcr[:H // 2, :W // 2].astype(np.uint8))
    return dict(sample=sample, recon=recon, modes=(lmodes, cmodes, pcm), report=report)


def set_idr_pic_id(sample: bytes, index: int) -> bytes:
    """Sample `index` of a stream: idr_pic_id 1 on even indices, 2 on odd ones (byte 6: 0x82 -> 0x83)."""
    if index % 2 == 0:
        return sample
    s = bytearray(sample)
    assert s[4] == 0x65 and s[6] == 0x82
    s[6] = 0x83
    return bytes(s)


# ---- MP4 (ISO/IEC 14496-12 and -15) ------------------------------------------------------------------------------
def box(kind: bytes, *payload: bytes) -> bytes:
    body = b"".join(payload)
    return struct.pack(">I", 8 + len(body)) + kind + body


def full_box(kind: bytes, version: int, flags: int, *payload: bytes) -> bytes:
    return box(kind, struct.pack(">I", (version << 24) | flags), *payload)


MATRIX = struct.pack(">9I", 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)


def moov(sizes, first_offset: int, width: int, height: int, qp: int, fps_num: int, fps_den: int) -> bytes:
    """The movie box of samples of `sizes` bytes stored back to back from file offset `first_offset`, one chunk each."""
    n = len(sizes)
    dur = n * fps_den
    sps, pps = parameter_sets(width, height, qp, fps_num, fps_den)
    avcc = box(b"avcC", bytes([1, sps[1], sps[2], sps[3], 0xFF, 0xE1]), struct.pack(">H", len(sps)), sps,
               bytes([1]), struct.pack(">H", len(pps)), pps)
    avc1 = box(b"avc1", bytes(6), struct.pack(">H", 1), bytes(16), struct.pack(">HH", width, height),
               struct.pack(">II", 0x480000, 0x480000), bytes(4), struct.pack(">H", 1), bytes(32),
               struct.pack(">Hh", 0x18, -1), avcc)
    offs = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])[:-1] + first_offset
    if n and int(offs[-1]) >= 2 ** 32:
        co = full_box(b"co64", 0, 0, struct.pack(">I", n), b"".join(struct.pack(">Q", int(o)) for o in offs))
    else:
        co = full_box(b"stco", 0, 0, struct.pack(">I", n), b"".join(struct.pack(">I", int(o)) for o in offs))
    stbl = box(b"stbl", full_box(b"stsd", 0, 0, struct.pack(">I", 1), avc1),
               full_box(b"stts", 0, 0, struct.pack(">III", 1, n, fps_den) if n else struct.pack(">I", 0)),
               full_box(b"stsc", 0, 0, struct.pack(">IIII", 1, 1, 1, 1)),
               full_box(b"stsz", 0, 0, struct.pack(">II", 0, n), b"".join(struct.pack(">I", int(s)) for s in sizes)),
               co)
    minf = box(b"minf", full_box(b"vmhd", 0, 1, bytes(8)),
               box(b"dinf", full_box(b"dref", 0, 0, struct.pack(">I", 1), full_box(b"url ", 0, 1))), stbl)
    mdia = box(b"mdia", full_box(b"mdhd", 0, 0, struct.pack(">IIIIHH", 0, 0, fps_num, dur, 0x55C4, 0)),
               full_box(b"hdlr", 0, 0, bytes(4), b"vide", bytes(12), b"VideoHandler\x00"), minf)
    tkhd = full_box(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, 1, 0, dur), bytes(8), struct.pack(">hhHH", 0, 0, 0, 0),
                    MATRIX, struct.pack(">II", width << 16, height << 16))
    mvhd = full_box(b"mvhd", 0, 0, struct.pack(">IIII", 0, 0, fps_num, dur), struct.pack(">IH", 0x10000, 0x100),
                    bytes(10), MATRIX, bytes(24), struct.pack(">I", 2))
    return box(b"moov", mvhd, box(b"trak", tkhd, mdia))


FTYP = box(b"ftyp", b"isom", struct.pack(">I", 512), b"isomiso2avc1mp41")


def mp4(samples, width: int, height: int, qp: int, fps_num: int = 25, fps_den: int = 1) -> bytes:
    """ftyp | mdat (64-bit largesize) | moov, the samples given with idr_pic_id 1 and set alternately here."""
    data = b"".join(set_idr_pic_id(s, i) for i, s in enumerate(samples))
    mdat = struct.pack(">I4sQ", 1, b"mdat", 16 + len(data)) + data
    return FTYP + mdat + moov([len(s) for s in samples], len(FTYP) + 16, width, height, qp, fps_num, fps_den)
