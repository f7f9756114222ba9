"""A plain restatement of the deblocked H.264 stream (csrc/h264.cu gab200_h264_encode_deblocked), written from ITU-T
H.264 clause 8.7 on top of tests/h264_stream_oracle.py, which it reuses unchanged -- what
tests/test_gpu_video_deblock.py compares the device's bytes with, and what FFmpeg's decoder referees in
tests/test_oracle_h264_deblock.py.

    frames = encode_stream(rgbs, qp, gop)   # [dict(sample, recon, filtered, types, mvs, report, paths), ...]
    data = mp4([f["sample"] for f in frames], W, H, qp, gop=gop)

The stream is tests/h264_stream_oracle.py's with two differences:

  * every slice header codes disable_deblocking_filter_idc 0 and slice_alpha_c0_offset_div2 =
    slice_beta_offset_div2 = 0 (ue(0) se(0) se(0) = 111 in place of ue(1) = 010, so nothing after it moves);
  * a P picture refers to the previous picture after the filter.  Intra prediction inside a picture still reads the
    picture's samples before the filter (8.3.1.2), so each frame has two pictures: `recon`, unfiltered, and
    `filtered`, the decoder's output and the next picture's reference.

The filter runs macroblock by macroblock in raster order: the luma vertical edges x = 0, 4, 8, 12 left to right, then
the horizontal edges y = 0, 4, 8, 12 top to bottom, and the same for Cb and Cr with edges 0 and 4; no left edge at
mbx 0 and no top edge at mby 0.  bS (8.7.2.1) per 4-sample segment: 4 on a macroblock edge with an intra side (I_16x16
or I_PCM), 3 on an intra macroblock's inner edge, 2 when either 4x4 luma block has coefficients, 1 when the two
vectors differ by 4 or more quarter samples in x or y, else 0; a chroma line takes the bS of the luma line twice its
index.  qP is the stream QP, 0 on an I_PCM side; chroma averages each side's QPc (Table 8-15).  `paths` counts, per
edge line, which way the filter went (tests/test_oracle_h264_deblock.py asserts the corpus reaches every one).
"""
from __future__ import annotations

from collections import Counter

import numpy as np

from oracle import h264 as O
from tests import h264_stream_oracle as S

# Table 8-16: alpha' and beta' by indexA = indexB = qPav (filter offsets 0)
ALPHA = [0] * 16 + [4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90,
                    101, 113, 127, 144, 162, 182, 203, 226, 255, 255]
BETA = [0] * 16 + [2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15,
                   15, 16, 16, 17, 17, 18, 18]
# Table 8-17: tC0 by indexA for bS = 1, 2, 3
TC0 = [(0, 0, 0)] * 17 + [(0, 0, 1), (0, 0, 1), (0, 0, 1), (0, 0, 1), (0, 1, 1), (0, 1, 1), (1, 1, 1), (1, 1, 1),
                          (1, 1, 1), (1, 1, 1), (1, 1, 2), (1, 1, 2), (1, 1, 2), (1, 1, 2), (1, 2, 3), (1, 2, 3),
                          (2, 2, 3), (2, 2, 4), (2, 3, 4), (2, 3, 4), (3, 3, 5), (3, 4, 6), (3, 4, 6), (4, 5, 7),
                          (4, 5, 8), (4, 6, 9), (5, 7, 10), (6, 8, 11), (6, 8, 13), (7, 10, 14), (8, 11, 16),
                          (9, 12, 18), (10, 13, 20), (11, 15, 23), (13, 17, 25)]
assert len(ALPHA) == len(BETA) == len(TC0) == 52
INTRA = ("I", "PCM")


def filter_lines(L, bS, qpav: int, chroma: bool, paths: Counter, kind: str):
    """One edge (8.7.2.2-8.7.2.4) on n lines across it: L (n, 8) int64 holds p3 p2 p1 p0 q0 q1 q2 q3 per line
    (chroma reads only p1 .. q1), bS (n,) the lines' strengths, all > 0; returns the filtered lines."""
    a, b = ALPHA[qpav], BETA[qpav]
    p3, p2, p1, p0, q0, q1, q2, q3 = (L[:, i].copy() for i in range(8))
    fa = np.abs(p0 - q0) < a
    fb = (np.abs(p1 - p0) < b) & (np.abs(q1 - q0) < b)
    on = fa & fb
    paths[(kind, "alpha_off")] += int(np.sum(~fa))
    paths[(kind, "beta_off")] += int(np.sum(fa & ~fb))
    out = L.copy()
    weak = on & (bS < 4)
    tc0 = np.array([TC0[qpav][min(max(int(s), 1), 3) - 1] for s in bS], np.int64)
    ap, aq = np.abs(p2 - p0) < b, np.abs(q2 - q0) < b
    if weak.any():
        tc = tc0 + 1 if chroma else tc0 + ap + aq
        raw = (((q0 - p0) << 2) + (p1 - q1) + 4) >> 3
        d = np.clip(raw, -tc, tc)
        paths[(kind, "tc_clip", "+")] += int(np.sum(weak & (raw > tc)))
        paths[(kind, "tc_clip", "-")] += int(np.sum(weak & (raw < -tc)))
        out[weak, 3] = np.clip(p0 + d, 0, 255)[weak]
        out[weak, 4] = np.clip(q0 - d, 0, 255)[weak]
        if not chroma:
            mid = (p0 + q0 + 1) >> 1
            wp, wq = weak & ap, weak & aq
            out[wp, 2] = (p1 + np.clip((p2 + mid - (p1 << 1)) >> 1, -tc0, tc0))[wp]
            out[wq, 5] = (q1 + np.clip((q2 + mid - (q1 << 1)) >> 1, -tc0, tc0))[wq]
            paths[(kind, "ap_only")] += int(np.sum(weak & ap & ~aq))
            paths[(kind, "aq_only")] += int(np.sum(weak & aq & ~ap))
        paths[(kind, "weak")] += int(np.sum(weak))
    strong4 = on & (bS == 4)
    if strong4.any():
        if chroma:
            out[strong4, 3] = ((2 * p1 + p0 + q1 + 2) >> 2)[strong4]
            out[strong4, 4] = ((2 * q1 + q0 + p1 + 2) >> 2)[strong4]
            paths[(kind, "bs4")] += int(np.sum(strong4))
        else:
            near = np.abs(p0 - q0) < ((a >> 2) + 2)
            sp, sq = strong4 & ap & near, strong4 & aq & near
            wp, wq = strong4 & ~(ap & near), strong4 & ~(aq & near)
            out[sp, 3] = ((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3)[sp]
            out[sp, 2] = ((p2 + p1 + p0 + q0 + 2) >> 2)[sp]
            out[sp, 1] = ((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3)[sp]
            out[wp, 3] = ((2 * p1 + p0 + q1 + 2) >> 2)[wp]
            out[sq, 4] = ((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3)[sq]
            out[sq, 5] = ((p0 + q0 + q1 + q2 + 2) >> 2)[sq]
            out[sq, 6] = ((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3)[sq]
            out[wq, 4] = ((2 * q1 + q0 + p1 + 2) >> 2)[wq]
            paths[(kind, "strong")] += int(np.sum(sp) + np.sum(sq))
            paths[(kind, "bs4_weak")] += int(np.sum(wp) + np.sum(wq))
    return out


def boundary_strength(types, mvs, totals, x, y, vertical: bool, e: int, seg: int, paths: Counter) -> int:
    """bS of segment seg (4 luma lines) of edge e (0: the macroblock edge) of macroblock (x, y)."""
    qx, qy = (e, seg) if vertical else (seg, e)
    if e:
        nx, ny = x, y
        px, py = (e - 1, seg) if vertical else (seg, e - 1)
    else:
        nx, ny = (x - 1, y) if vertical else (x, y - 1)
        px, py = (3, seg) if vertical else (seg, 3)
    tq, tp = types[y, x], types[ny, nx]
    if tq in INTRA or tp in INTRA:
        return 3 if e else 4
    if totals[4 * y + qy, 4 * x + qx] or totals[4 * ny + py, 4 * nx + px]:
        return 2
    d = np.abs(mvs[y, x] - mvs[ny, nx])
    for axis, v in zip("xy", d):
        if v in (3, 4):
            paths[("mv_diff", axis, int(v))] += 1
    return 1 if (d >= 4).any() else 0


def deblock(recon, types, mvs, totals, qp: int, is_p: bool = False):
    """8.7 on a picture: recon = padded (Y, Cb, Cr) before the filter, types (hm, wm) 'I', 'PCM', 'P' or 'P_Skip',
    mvs (hm, wm, 2) quarter samples, totals (4 hm, 4 wm) the luma 4x4 blocks' TotalCoeff.  Returns ((Y, Cb, Cr)
    filtered, Counter of the paths taken)."""
    planes = [np.asarray(p, np.int64).copy() for p in recon]
    hm, wm = types.shape
    paths = Counter()
    qpc = O.CHROMA_QP
    for y in range(hm):
        for x in range(wm):
            qq = 0 if types[y, x] == "PCM" else qp
            if x == 0:
                paths[("border", "left")] += 1
            if y == 0:
                paths[("border", "top")] += 1
            for vertical in (True, False):
                has = x > 0 if vertical else y > 0
                nb = (types[y, x - 1] if vertical else types[y - 1, x]) if has else None
                qn = 0 if nb == "PCM" else qp
                bs = np.zeros((4, 4), np.int64)
                for e in range(4):
                    if e == 0 and not has:
                        continue
                    for seg in range(4):
                        bs[e, seg] = boundary_strength(types, mvs, totals, x, y, vertical, e, seg, paths)
                if has and (qq == 0) != (qn == 0):
                    paths[("pcm_edge",)] += 1
                if is_p and types[y, x] in INTRA:
                    paths[("intra_in_p",)] += 1
                for p, plane in enumerate(planes):
                    n = 16 if p == 0 else 8
                    for e in range(4 if p == 0 else 2):
                        edge = e if p == 0 else 2 * e       # the luma edge a chroma edge takes its bS from
                        if edge == 0 and not has:
                            continue
                        line_bs = np.repeat(bs[edge], 4 if p == 0 else 2)
                        kind = "luma" if p == 0 else "chroma"
                        for v in np.unique(line_bs):
                            paths[(kind, "bS", int(v))] += int(np.sum(line_bs == v))
                        if p == 0:
                            qpav = (qq + qn + 1) >> 1 if edge == 0 else qq
                        else:
                            qpav = (qpc[qq] + qpc[qn] + 1) >> 1 if edge == 0 else qpc[qq]
                        sel = line_bs > 0
                        if not sel.any():
                            continue
                        c0 = n * (x if vertical else y) + 4 * e          # q0's coordinate across the edge
                        lines = np.arange(n) + n * (y if vertical else x)
                        idx = c0 + np.arange(-4, 4)
                        L = plane[lines[:, None], idx[None, :]] if vertical else plane[idx[None, :], lines[:, None]]
                        F = filter_lines(L[sel], line_bs[sel], qpav, p > 0, paths, kind)
                        L[sel] = F
                        if vertical:
                            plane[lines[:, None], idx[None, :]] = L
                        else:
                            plane[idx[None, :], lines[:, None]] = L
    return tuple(p.astype(np.uint8) for p in planes), paths


def deblocked_sample(sample: bytes) -> bytes:
    """The sample with disable_deblocking_filter_idc 0 and both offsets se(0): the slice header's last three bits
    010 -> 111 (bits 19-21 of an IDR slice's RBSP, 15-17 of a P slice's; the bytes around them are never zero, so
    emulation prevention does not move)."""
    s = bytearray(sample)
    if s[4] == 0x65:
        assert s[7] & 0x1C == 0x08
        s[7] |= 0x14
    else:
        assert s[4] == 0x61 and s[6] & 1 == 0 and s[7] & 0xC0 == 0x80
        s[6] |= 0x01
        s[7] |= 0x40
    return bytes(s)


def _encode_with_totals(encode, *args):
    """encode(*args) and the (4 hm, 4 wm) TotalCoeff grid its P_L0_16x16 macroblocks' levels filled in (zeros when
    it coded none), taken from the grid tests/h264_stream_oracle.inter_residual_bits writes into."""
    grids = []
    orig = S.inter_residual_bits

    def capture(mx, my, lev, cdcl, cacl, tl_, tc_, report):
        grids[:] = [tl_]
        return orig(mx, my, lev, cdcl, cacl, tl_, tc_, report)

    S.inter_residual_bits = capture
    try:
        f = encode(*args)
    finally:
        S.inter_residual_bits = orig
    hm, wm = f["types"].shape
    return f, grids[0] if grids else np.zeros((4 * hm, 4 * wm), np.int64)


def encode_stream(frames, qp: int, gop: int, start: int = 0, ref=None) -> list:
    """tests/h264_stream_oracle.encode_stream's frames, deblocked: per frame dict(sample, recon (unfiltered, padded),
    filtered (padded, the decoder's output), types, mvs, report, paths).  ref: the filtered picture before frames[0]
    (when start % gop)."""
    if not 1 <= gop <= 65535:
        raise ValueError(f"gop must be in 1..65535, got {gop}")
    out = []
    for k, rgb in enumerate(frames):
        n = start + k
        if n % gop == 0:
            f, totals = _encode_with_totals(S.encode_idr, rgb, qp)
        else:
            f, totals = _encode_with_totals(S.encode_p, rgb, qp, ref, (n % gop) % 16)
            f["report"].add(("frame_num", (n % gop) % 16))
        f["filtered"], f["paths"] = deblock(f["recon"], f["types"], f["mvs"], totals, qp, n % gop != 0)
        f["sample"] = deblocked_sample(f["sample"])
        ref = f["filtered"]
        out.append(f)
    return out


crop = S.crop
# the parameter sets and the container are the same with and without the filter
mp4 = S.mp4
