"""A plain restatement of the device H.264 stream encode with P pictures (csrc/h264.cu gab200_h264_encode_stream),
written from ITU-T H.264 clauses 7.3.4, 7.3.5, 8.4 and 9.2 on top of oracle/h264.py's intra coding, which it reuses
unchanged -- what tests/test_gpu_video_gop.py compares the device's bytes with, and what FFmpeg's decoder referees in
tests/test_oracle_h264_inter.py.

    frames = encode_stream(rgbs, qp, gop)   # [dict(sample, recon=(Y, Cb, Cr) padded, types, mvs, report), ...]
    data = mp4([f["sample"] for f in frames], W, H, qp, gop=gop)

The stream: stream position n is an IDR picture when n % gop == 0 (byte for byte oracle.h264.encode_frame's sample),
otherwise one P slice that refers to the previous picture.  Each P macroblock is decided from pixels alone:

  * an integer full search over +-16 samples around (0, 0) by 16x16 luma SAD + lambda * (se(v) bits of the vector's
    two components in quarter samples), then a half-sample and a quarter-sample refinement over the 8 neighbours by
    SATD + the same term; every minimum keeps the first candidate in its order (raster for the full search, the
    centre first for a refinement);
  * intra (I_16x16, oracle/h264.py's mode decision) when its least luma SATD + INTRA_BIAS * lambda is below the inter
    cost, otherwise P_L0_16x16;
  * inter residuals quantised with the dead zone f = 2^qbits / 6, luma as sixteen 16-coefficient 4x4 blocks;
  * I_PCM when a level falls outside +-2063 or the macroblock's bits, the motion vector difference and the skip run
    aside, exceed I_PCM's 9 + 3072.

Only then are the motion-vector predictors (8.4.1.3), the P_Skip predictors (8.4.1.1) and the skip runs derived: a
P_L0_16x16 macroblock with no coded coefficient whose vector equals its mvpSkip is P_Skip.  The reference is the
previous picture's whole padded reconstruction, its samples read at coordinates clamped to the coded picture.
"""
from __future__ import annotations

import struct

import numpy as np

from oracle import h264 as O

SEARCH = 16                  # integer search range, samples
INTRA_BIAS = 24              # intra's SATD handicap, in units of lambda
P_HEADER_BITS = 18           # the P slice header after the NAL header byte (see p_slice_header)
MVD_BITS = 2 * 17            # se(v) of the largest |mvd| (2 * 67 quarter samples) in each component
# Table 9-4, inter column: coded_block_pattern -> codeNum
INTER_CBP_CODE = [0] * 48
for _k, _c in enumerate([0, 16, 1, 2, 4, 8, 32, 3, 5, 10, 12, 15, 47, 7, 11, 13, 14, 6, 9, 31, 35, 37, 42, 44, 33, 34,
                         36, 40, 39, 43, 45, 46, 17, 18, 20, 24, 19, 21, 26, 28, 23, 27, 29, 30, 22, 25, 38, 41]):
    INTER_CBP_CODE[_c] = _k
NEIGHBOURS = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1)]   # (dy, dx), refinement order


def lam(qp: int) -> int:
    """The motion cost's lambda: 2^max(0, (qp - 12) // 6)."""
    return 1 << max(0, (qp - 12) // 6)


def ue_len(v):
    return 2 * np.floor(np.log2(np.asarray(v, np.float64) + 1)).astype(np.int64) + 1


def se_len(v):
    v = np.asarray(v, np.int64)
    return ue_len(np.where(v > 0, 2 * v - 1, -2 * v))


def p_bound(width: int, height: int) -> int:
    """The largest P sample of a width x height frame: 4 + 1 + n + ceil(n / 2) for the n bytes of a slice whose every
    macroblock carries a skip run of at most 3 bits per macroblock it closes, a motion vector difference of at most
    MVD_BITS and I_PCM at its worst alignment; -1 where oracle.h264.bound is -1."""
    if O.bound(width, height) < 0:
        return -1
    nmb = ((width + 15) // 16) * ((height + 15) // 16)
    n = (P_HEADER_BITS + nmb * (3 + MVD_BITS + O.PCM_BITS + 7) + 1 + 7) // 8
    return 5 + n + (n + 1) // 2


def parameter_sets(width, height, qp, fps_num=25, fps_den=1, gop=1):
    """oracle.h264.parameter_sets, with max_num_ref_frames 1 when gop > 1 (the one field that differs)."""
    sps, pps = O.parameter_sets(width, height, qp, fps_num, fps_den)
    if gop == 1:
        return sps, pps
    raw = _unescape(sps[1:])
    bits = bin(int.from_bytes(raw, "big"))[2:].zfill(8 * len(raw)).rstrip("0")[:-1]   # without rbsp_trailing_bits
    # profile, constraints and level (24 bits), then ue(0) ue(0) ue(2) ue(0): the last, max_num_ref_frames, -> ue(1)
    assert bits[24:30] == "110111"
    b = O.Bits()
    b.u(int(bits[:29] + "010" + bits[30:], 2), len(bits) + 2)
    return O.nal(7, O.to_bytes(O.rbsp_trailing(b))), pps


def _unescape(data: bytes) -> bytes:
    out, zeros = bytearray(), 0
    for x in data:
        if zeros >= 2 and x == 3:
            zeros = 0
            continue
        out.append(x)
        zeros = zeros + 1 if x == 0 else 0
    return bytes(out)


# ---- interpolation (8.4.2.2) ---------------------------------------------------------------------------------------
def _tap(a, b, c, d, e, f):
    return a - 5 * b + 20 * c + 20 * d - 5 * e + f


def luma_pred(ref, x, y, mvx, mvy):
    """8.4.2.2.1: the luma samples at integer positions (x, y) (arrays) displaced by quarter-sample vectors (mvx, mvy),
    the reference read at coordinates clamped to its (coded) size."""
    H, W = ref.shape
    ref = ref.astype(np.int64)
    xi, yi, xf, yf = x + (mvx >> 2), y + (mvy >> 2), mvx & 3, mvy & 3

    def G(dx, dy):
        return ref[np.clip(yi + dy, 0, H - 1), np.clip(xi + dx, 0, W - 1)]

    def hor(dy):
        return _tap(*(G(dx, dy) for dx in range(-2, 4)))

    def ver(dx):
        return _tap(*(G(dx, dy) for dy in range(-2, 4)))

    clip = lambda v, s, r: np.clip((v + r) >> s, 0, 255)       # noqa: E731
    g, hh, mm = G(0, 0), G(1, 0), G(0, 1)
    b, s = clip(hor(0), 5, 16), clip(hor(1), 5, 16)
    h1, m1 = ver(0), ver(1)
    h, m = clip(h1, 5, 16), clip(m1, 5, 16)
    j = clip(_tap(ver(-2), ver(-1), h1, m1, ver(2), ver(3)), 10, 512)
    avg = lambda p, q: (p + q + 1) >> 1                          # noqa: E731
    table = {(0, 0): g, (0, 1): avg(g, h), (0, 2): h, (0, 3): avg(mm, h), (1, 0): avg(g, b), (1, 1): avg(b, h),
             (1, 2): avg(h, j), (1, 3): avg(h, s), (2, 0): b, (2, 1): avg(b, j), (2, 2): j, (2, 3): avg(j, s),
             (3, 0): avg(hh, b), (3, 1): avg(b, m), (3, 2): avg(j, m), (3, 3): avg(m, s)}
    out = np.zeros(np.broadcast(xi, yi).shape, np.int64)
    for (fx, fy), v in table.items():
        sel = (xf == fx) & (yf == fy)
        out = np.where(sel, v, out)
    return out


def chroma_pred(ref, x, y, mvx, mvy):
    """8.4.2.2.2: chroma samples at (x, y) displaced by (mvx, mvy) in eighth samples, coordinates clamped."""
    H, W = ref.shape
    ref = ref.astype(np.int64)
    xi, yi, xf, yf = x + (mvx >> 3), y + (mvy >> 3), mvx & 7, mvy & 7

    def G(dx, dy):
        return ref[np.clip(yi + dy, 0, H - 1), np.clip(xi + dx, 0, W - 1)]

    return ((8 - xf) * (8 - yf) * G(0, 0) + xf * (8 - yf) * G(1, 0) + (8 - xf) * yf * G(0, 1) + xf * yf * G(1, 1)
            + 32) >> 6


def _mb_grid(hm, wm, n):
    """(hm, wm, n, n) x and y sample coordinates of every macroblock's n x n block."""
    my, mx = np.mgrid[0:hm, 0:wm]
    j, i = np.mgrid[0:n, 0:n]
    return (n * mx)[..., None, None] + i, (n * my)[..., None, None] + j


# ---- motion search -------------------------------------------------------------------------------------------------
def search(ys, ref_y, qp):
    """Every macroblock's vector (hm, wm, 2) [x, y] in quarter samples, its luma prediction (hm, wm, 16, 16) and its
    cost (hm, wm)."""
    hc, wc = ys.shape
    hm, wm = hc // 16, wc // 16
    L = lam(qp)
    src = ys.astype(np.int64)
    pad = np.pad(ref_y.astype(np.int64), SEARCH, mode="edge")
    best = np.full((hm, wm), np.iinfo(np.int64).max)
    bv = np.zeros((hm, wm, 2), np.int64)
    for dy in range(-SEARCH, SEARCH + 1):
        for dx in range(-SEARCH, SEARCH + 1):
            d = np.abs(src - pad[SEARCH + dy:SEARCH + dy + hc, SEARCH + dx:SEARCH + dx + wc])
            c = d.reshape(hm, 16, wm, 16).sum((1, 3)) + L * (se_len(4 * dx) + se_len(4 * dy))
            better = c < best
            best = np.where(better, c, best)
            bv[better] = (4 * dx, 4 * dy)
    X, Y = _mb_grid(hm, wm, 16)
    srcb = src.reshape(hm, 16, wm, 16).swapaxes(1, 2)

    def cost(v):
        p = luma_pred(ref_y, X, Y, v[..., 0, None, None], v[..., 1, None, None])
        return O.satd(srcb - p) + L * (se_len(v[..., 0]) + se_len(v[..., 1])), p

    for step in (2, 1):
        c0, p0 = cost(bv)
        nv = bv.copy()
        for dy, dx in NEIGHBOURS:
            v = bv + np.array([dx * step, dy * step])
            c, p = cost(v)
            better = c < c0
            c0 = np.where(better, c, c0)
            nv[better] = v[better]
        bv = nv
    c, p = cost(bv)
    return bv, p, c


# ---- inter transform and quantisation -------------------------------------------------------------------------------
def quant_inter(c, qp, mf, dc):
    qbits = 15 + qp // 6
    f = (1 << qbits) // 6
    q = (np.abs(c) * mf + 2 * f) >> (qbits + 1) if dc else (np.abs(c) * mf + f) >> qbits
    return np.sign(c) * q


def code_luma_inter(res, qp):
    """res (M, 16, 16) -> (levels (M, 4, 4, 4, 4) [block row, block column, raster], reconstructed residual)."""
    w = O.CF @ O.blocks(res) @ O.CF.T
    lev = quant_inter(w, qp, O.MF[qp % 6][O.POS], False)
    return lev, O.unblocks(O.idct4(O.dequant_ac(lev, qp)))


def code_chroma_inter(res, qpc):
    w = O.CF @ O.blocks(res) @ O.CF.T
    t = O.H2 @ w[..., 0, 0] @ O.H2
    dcl = quant_inter(t, qpc, O.MF[qpc % 6, 0], True)
    acl = quant_inter(w, qpc, O.MF[qpc % 6][O.POS], False)
    acl[..., 0, 0] = 0
    return dcl, acl, O.recon_chroma(dcl, acl, qpc)


# ---- macroblock bits (7.3.5) ----------------------------------------------------------------------------------------
def intra_bits(mx, my, lmode, cmode, dcl, acl, cdcl, cacl, tl_, tc_, report, offset):
    """oracle.h264.macroblock_bits with mb_type + offset (5 in a P slice)."""
    b = O.macroblock_bits(mx, my, lmode, cmode, dcl, acl, cdcl, cacl, tl_, tc_, report)
    if offset:
        cbpl = 15 if np.any(acl) else 0
        cbpc = 2 if np.any(cacl) else 1 if np.any(cdcl) else 0
        t = 1 + lmode + 4 * cbpc + (12 if cbpl else 0)
        old = O.Bits()
        old.ue(t)
        new = O.Bits()
        new.ue(t + offset)
        s = b.bits()
        assert s.startswith(old.bits())
        b = O.Bits()
        b.parts.append(new.bits() + s[old.n:])
        b.n = len(b.parts[0])
    return b


def inter_residual_bits(mx, my, lev, cdcl, cacl, tl_, tc_, report):
    """The P_L0_16x16 macroblock's coded_block_pattern, mb_qp_delta and residual bits (mvd excluded) and its cbp;
    fills its totals into the grids."""
    cbpl = 0
    for k in range(4):
        if np.any(lev[2 * (k // 2):2 * (k // 2) + 2, 2 * (k % 2):2 * (k % 2) + 2]):
            cbpl |= 1 << k
    cbpc = 2 if np.any(cacl) else 1 if np.any(cdcl) else 0
    for bx, by in O.LUMA_BLK:
        k8 = (by // 2) * 2 + bx // 2
        tl_[4 * my + by, 4 * mx + bx] = np.count_nonzero(lev[by, bx]) if (cbpl >> k8) & 1 else 0
    for c in range(2):
        for by in range(2):
            for bx in range(2):
                tc_[c][2 * my + by, 2 * mx + bx] = np.count_nonzero(cacl[c, by, bx]) if cbpc == 2 else 0
    cbp = cbpl | cbpc << 4
    b = O.Bits()
    b.ue(INTER_CBP_CODE[cbp])
    report.add(("inter_cbp", cbp))
    if cbp:
        b.se(0)
    for bx, by in O.LUMA_BLK:
        k8 = (by // 2) * 2 + bx // 2
        if (cbpl >> k8) & 1:
            n = O.residual_block(b, lev[by, bx].reshape(16)[O.ZIGZAG], O.nc_of(tl_, 4 * mx + bx, 4 * my + by), report)
            if n == 16:
                report.add(("luma_total", 16))
    if cbpc:
        for c in range(2):
            O.residual_block(b, cdcl[c].reshape(4), -1, report)
    if cbpc == 2:
        for c in range(2):
            for by in range(2):
                for bx in range(2):
                    O.residual_block(b, cacl[c, by, bx].reshape(16)[O.ZIGZAG[1:]],
                                     O.nc_of(tc_[c], 2 * mx + bx, 2 * my + by), report)
    return b, cbp


# ---- motion vector prediction (8.4.1.1, 8.4.1.3) --------------------------------------------------------------------
def predictors(types, mvs):
    """(mvp, mvpSkip), each (hm, wm, 2), from the macroblock types ('P', 'I' or 'PCM') and vectors."""
    hm, wm = types.shape
    mvp = np.zeros((hm, wm, 2), np.int64)
    skip = np.zeros((hm, wm, 2), np.int64)
    for y in range(hm):
        for x in range(wm):
            def nb(xx, yy):
                if not (0 <= xx < wm and 0 <= yy < hm):
                    return None
                return (0, tuple(mvs[yy, xx])) if types[yy, xx] == "P" else (-1, (0, 0))

            A, B, C = nb(x - 1, y), nb(x, y - 1), nb(x + 1, y - 1)
            if C is None:
                C = nb(x - 1, y - 1)
            availA = A is not None
            A = A or (-1, (0, 0))
            if B is None and C is None and availA:
                B = C = A
            B = B or (-1, (0, 0))
            C = C or (-1, (0, 0))
            match = [n for n in (A, B, C) if n[0] == 0]
            if len(match) == 1:
                p = match[0][1]
            else:
                p = tuple(sorted([A[1][k], B[1][k], C[1][k]])[1] for k in range(2))
            mvp[y, x] = p
            a, b = nb(x - 1, y), nb(x, y - 1)
            if a is None or b is None or a == (0, (0, 0)) or b == (0, (0, 0)):
                skip[y, x] = (0, 0)
            else:
                skip[y, x] = p
    return mvp, skip


# ---- slice headers --------------------------------------------------------------------------------------------------
def p_slice_header(b, frame_num: int):
    b.ue(0)                          # first_mb_in_slice
    b.ue(5)                          # slice_type: P (all slices of the picture)
    b.ue(0)                          # pic_parameter_set_id
    b.u(frame_num, 4)
    b.u(0, 1)                        # num_ref_idx_active_override_flag
    b.u(0, 1)                        # ref_pic_list_modification_flag_l0
    b.u(0, 1)                        # adaptive_ref_pic_marking_mode_flag
    b.se(0)                          # slice_qp_delta
    b.ue(1)                          # disable_deblocking_filter_idc


# ---- the encode -----------------------------------------------------------------------------------------------------
def _pcm_bits(pos, ys, cbs, crs, x, y):
    head = "000011111" + "0" * (-(pos + 9) % 8)             # ue(30), pcm_alignment_zero_bits
    samples = np.concatenate([ys[16 * y:16 * y + 16, 16 * x:16 * x + 16].ravel(),
                              cbs[8 * y:8 * y + 8, 8 * x:8 * x + 8].ravel(),
                              crs[8 * y:8 * y + 8, 8 * x:8 * x + 8].ravel()])
    return head + "".join(format(int(v), "08b") for v in samples)


def encode_p(rgb, qp, ref, frame_num):
    """One P picture of rgb against the padded reconstruction ref = (Y, Cb, Cr) of the previous picture; with ref
    None, the IDR picture's padded reconstruction and macroblock types (its sample is oracle.h264.encode_frame's)."""
    rgb = np.asarray(rgb, np.uint8)
    H, W, _ = rgb.shape
    qpc = O.CHROMA_QP[qp]
    ys, cbs, crs = O.rgb_to_yuv(rgb)
    hc, wc = ys.shape
    hm, wm = hc // 16, wc // 16
    report = set()
    if ref is None:                                # intra only: the inter candidate never wins
        mv, ipred = np.zeros((hm, wm, 2), np.int64), np.zeros((hm, wm, 16, 16), np.int64)
        icost = np.full((hm, wm), np.iinfo(np.int64).max)
        cpred = [np.zeros((hm, wm, 8, 8), np.int64)] * 2
    else:
        mv, ipred, icost = search(ys, ref[0], qp)
        X, Y = _mb_grid(hm, wm, 8)
        cpred = [chroma_pred(r, X, Y, mv[..., 0, None, None], mv[..., 1, None, None]) for r in ref[1:]]
    L = lam(qp)
    ry, rcb, rcr = np.zeros_like(ys), np.zeros_like(cbs), np.zeros_like(crs)
    tl_ = np.zeros((4 * hm, 4 * wm), np.int64)
    tc_ = [np.zeros((2 * hm, 2 * wm), np.int64) for _ in range(2)]
    types = np.full((hm, wm), "P", dtype=object)
    cbps = np.zeros((hm, wm), np.int64)
    mbbits = {}
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
        pl = O.predict(top, left, tlv, has_t, has_l, 16, False)
        lav = np.stack([has_t, has_l, np.ones(M, bool), has_t & has_l], 1)
        lcost = np.where(lav, O.satd(src[:, None] - pl), np.iinfo(np.int64).max)
        lm = np.argmin(lcost, 1)
        intra = lcost[np.arange(M), lm] + INTRA_BIAS * L < icost[my, mx]
        cy = (8 * my)[:, None] + np.arange(8)
        cx = (8 * mx)[:, None] + np.arange(8)
        csrc, cpa = [], []
        for plane, rp in ((cbs, rcb), (crs, rcr)):
            csrc.append(plane[cy[:, :, None], cx[:, None, :]])
            top = np.where(has_t[:, None], rp[np.maximum(8 * my - 1, 0)[:, None], cx], 0)
            left = np.where(has_l[:, None], rp[cy, np.maximum(8 * mx - 1, 0)[:, None]], 0)
            tlv = np.where(has_t & has_l, rp[np.maximum(8 * my - 1, 0), np.maximum(8 * mx - 1, 0)], 0)
            cpa.append(O.predict(top, left, tlv, has_t, has_l, 8, True))
        cav = np.stack([np.ones(M, bool), has_l, has_t, has_t & has_l], 1)
        cm = O.choose(cpa, csrc, cav)
        # intra candidates
        lp = pl[np.arange(M), lm]
        dcl, acl, rres = O.code_luma(src - lp, qp)
        ires = [O.code_chroma(s - p[np.arange(M), cm], qpc) for s, p in zip(csrc, cpa)]
        # inter candidates
        ip = ipred[my, mx]
        lev, pres = code_luma_inter(src - ip, qp)
        cp = [c[my, mx] for c in cpred]
        pres_c = [code_chroma_inter(s - p, qpc) for s, p in zip(csrc, cp)]
        for i in range(M):
            x, y = int(mx[i]), int(my[i])
            b = None
            if intra[i]:
                cdcl = np.stack([r[0][i] for r in ires])
                cacl = np.stack([r[1][i] for r in ires])
                over = max(np.abs(dcl[i]).max(), np.abs(acl[i]).max(), np.abs(cdcl).max(), np.abs(cacl).max())
                if over <= O.MAX_LEVEL:
                    rep = set()
                    b = intra_bits(x, y, int(lm[i]), int(cm[i]), dcl[i], acl[i], cdcl, cacl, tl_, tc_, rep,
                                   0 if ref is None else 5)
                    if b.n <= O.PCM_BITS:
                        report |= rep
                        types[y, x] = "I"
                        report.add(("mb", "I_16x16"))
                        ry[16 * y:16 * y + 16, 16 * x:16 * x + 16] = np.clip(lp[i] + rres[i], 0, 255)
                        for k, rp in enumerate((rcb, rcr)):
                            rp[8 * y:8 * y + 8, 8 * x:8 * x + 8] = np.clip(cpa[k][i, cm[i]] + ires[k][2][i], 0, 255)
                    else:
                        b = None
            else:
                cdcl = np.stack([r[0][i] for r in pres_c])
                cacl = np.stack([r[1][i] for r in pres_c])
                over = max(np.abs(lev[i]).max(), np.abs(cdcl).max(), np.abs(cacl).max())
                if over <= O.MAX_LEVEL:
                    rep = set()
                    rb, cbp = inter_residual_bits(x, y, lev[i], cdcl, cacl, tl_, tc_, rep)
                    if 1 + rb.n <= O.PCM_BITS:
                        b = rb
                        report |= rep
                        cbps[y, x] = cbp
                        ry[16 * y:16 * y + 16, 16 * x:16 * x + 16] = np.clip(ip[i] + pres[i], 0, 255)
                        for k, rp in enumerate((rcb, rcr)):
                            rp[8 * y:8 * y + 8, 8 * x:8 * x + 8] = np.clip(cp[k][i] + pres_c[k][2][i], 0, 255)
            if b is None:
                types[y, x] = "PCM"
                report.add(("mb", "I_PCM"))
                tl_[4 * y:4 * y + 4, 4 * x:4 * x + 4] = 16
                for t in tc_:
                    t[2 * y:2 * y + 2, 2 * x:2 * x + 2] = 16
                ry[16 * y:16 * y + 16, 16 * x:16 * x + 16] = src[i]
                rcb[8 * y:8 * y + 8, 8 * x:8 * x + 8] = csrc[0][i]
                rcr[8 * y:8 * y + 8, 8 * x:8 * x + 8] = csrc[1][i]
            else:
                mbbits[(y, x)] = b.bits()
    if ref is None:
        out = O.encode_frame(rgb, qp)
        assert all(np.array_equal(a, b) for a, b in zip(out["recon"], crop((ry, rcb, rcr), W, H)))
        return dict(sample=out["sample"], recon=(ry, rcb, rcr), types=types, mvs=np.zeros_like(mv),
                    report=out["report"])
    mvs = np.where((types == "P")[..., None], mv, 0)
    mvp, mvps = predictors(types, mvs)
    skipped = (types == "P") & (cbps == 0) & np.all(mvs == mvps, -1)
    b = O.Bits()
    p_slice_header(b, frame_num)
    assert b.n == P_HEADER_BITS
    parts, n, run = [b.bits()], b.n, 0
    for y in range(hm):
        for x in range(wm):
            if skipped[y, x]:
                run += 1
                continue
            r = O.Bits()
            r.ue(run)
            report.add(("mb_skip_run", "0" if run == 0 else "mid"))
            run = 0
            if types[y, x] == "PCM":
                s = r.bits() + _pcm_bits(n + r.n, ys, cbs, crs, x, y)
            elif types[y, x] == "I":
                s = r.bits() + mbbits[(y, x)]
            else:
                m = O.Bits()
                m.ue(0)                                      # mb_type P_L0_16x16
                dv = mvs[y, x] - mvp[y, x]
                m.se(int(dv[0]))
                m.se(int(dv[1]))
                for v in dv:
                    report.add(("mvd", "0" if v == 0 else "1" if abs(v) == 1 else "other"))
                report.add(("mb", "P_L0_16x16"))
                s = r.bits() + m.bits() + mbbits[(y, x)]
            parts.append(s)
            n += len(s)
    if run:
        r = O.Bits()
        r.ue(run)
        parts.append(r.bits())
        report.add(("mb_skip_run", "all" if run == hm * wm else "trailing"))
    if skipped.any():
        report.add(("mb", "P_Skip"))
    parts.append("1")
    rbsp = O.to_bytes("".join(parts))
    esc, inserted = O.emulation_prevention(rbsp)
    if inserted:
        report.add(("emulation_prevention",))
    body = b"\x61" + esc
    sample = struct.pack(">I", len(body)) + body
    assert len(sample) <= p_bound(W, H)
    t = np.where(skipped, "P_Skip", types)
    for v in np.unique(mvs[types == "P"] & 3):
        report.add(("mv_frac", int(v)))
    my, mx = np.nonzero(types == "P")
    vx, vy = mvs[my, mx, 0], mvs[my, mx, 1]
    for side, hit in (("left", 16 * mx + (vx >> 2) < 0), ("right", 16 * mx + 16 + ((vx + 3) >> 2) > wc),
                      ("top", 16 * my + (vy >> 2) < 0), ("bottom", 16 * my + 16 + ((vy + 3) >> 2) > hc)):
        if hit.any():
            report.add(("outside", side))
    if np.any(np.abs(mvs - mvp)[~skipped & (types == "P")] >= 64):
        report.add(("mvd_extreme",))
    return dict(sample=sample, recon=(ry, rcb, rcr), types=t, mvs=mvs, report=report)


def encode_idr(rgb, qp):
    """oracle.h264.encode_frame's sample, with the padded reconstruction the P pictures after it refer to."""
    return encode_p(rgb, qp, None, 0)


def encode_stream(frames, qp: int, gop: int, start: int = 0, ref=None) -> list:
    """Per frame dict(sample, recon: padded (Y, Cb, Cr), types: (hm, wm) 'I', 'PCM', 'P' or 'P_Skip', mvs (hm, wm, 2),
    report).  start: the stream position of frames[0]; ref: the padded reconstruction before it (when start % gop)."""
    if not 1 <= gop <= 65535:
        raise ValueError(f"gop must be in 1..65535, got {gop}")
    out = []
    for k, rgb in enumerate(frames):
        n = start + k
        if n % gop == 0:
            f = encode_idr(rgb, qp)
        else:
            f = encode_p(rgb, qp, ref, (n % gop) % 16)
            f["report"].add(("frame_num", (n % gop) % 16))
        ref = f["recon"]
        out.append(f)
    return out


def crop(recon, W, H):
    return recon[0][:H, :W].astype(np.uint8), recon[1][:H // 2, :W // 2].astype(np.uint8), \
        recon[2][:H // 2, :W // 2].astype(np.uint8)


# ---- MP4 ------------------------------------------------------------------------------------------------------------
def set_idr_pic_id(samples) -> list:
    """idr_pic_id 2 on the odd-numbered IDR samples (byte 6: 0x82 -> 0x83)."""
    out, k = [], 0
    for s in samples:
        if s[4] == 0x65:
            if k % 2:
                s = bytearray(s)
                assert s[6] == 0x82
                s[6] = 0x83
                s = bytes(s)
            k += 1
        out.append(s)
    return out


def mp4(samples, width, height, qp, fps_num=25, fps_den=1, gop=1) -> bytes:
    """oracle.h264.mp4 with max_num_ref_frames 1 and an stss box listing the IDR samples (1-based) when gop > 1."""
    if gop == 1:
        return O.mp4(samples, width, height, qp, fps_num, fps_den)
    samples = set_idr_pic_id(samples)
    data = b"".join(samples)
    mdat = struct.pack(">I4sQ", 1, b"mdat", 16 + len(data)) + data
    return O.FTYP + mdat + moov([len(s) for s in samples], [s[4] == 0x65 for s in samples], len(O.FTYP) + 16, width,
                                height, qp, fps_num, fps_den, gop)


def moov(sizes, sync, first_offset, width, height, qp, fps_num, fps_den, gop) -> bytes:
    """oracle.h264.moov with this stream's SPS, and stss after stsz when gop > 1."""
    n = len(sizes)
    dur = n * fps_den
    sps, pps = parameter_sets(width, height, qp, fps_num, fps_den, gop)
    avcc = O.box(b"avcC", bytes([1, sps[1], sps[2], sps[3], 0xFF, 0xE1]), struct.pack(">H", len(sps)), sps,
                 bytes([1]), struct.pack(">H", len(pps)), pps)
    avc1 = O.box(b"avc1", bytes(6), struct.pack(">H", 1), bytes(16), struct.pack(">HH", width, height),
                 struct.pack(">II", 0x480000, 0x480000), bytes(4), struct.pack(">H", 1), bytes(32),
                 struct.pack(">Hh", 0x18, -1), avcc)
    offs = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])[:-1] + first_offset
    if n and int(offs[-1]) >= 2 ** 32:
        co = O.full_box(b"co64", 0, 0, struct.pack(">I", n), b"".join(struct.pack(">Q", int(o)) for o in offs))
    else:
        co = O.full_box(b"stco", 0, 0, struct.pack(">I", n), b"".join(struct.pack(">I", int(o)) for o in offs))
    ids = [i + 1 for i, s in enumerate(sync) if s]
    stss = O.full_box(b"stss", 0, 0, struct.pack(">I", len(ids)), b"".join(struct.pack(">I", i) for i in ids)) \
        if gop > 1 else b""
    stbl = O.box(b"stbl", O.full_box(b"stsd", 0, 0, struct.pack(">I", 1), avc1),
                 O.full_box(b"stts", 0, 0, struct.pack(">III", 1, n, fps_den) if n else struct.pack(">I", 0)),
                 O.full_box(b"stsc", 0, 0, struct.pack(">IIII", 1, 1, 1, 1)),
                 O.full_box(b"stsz", 0, 0, struct.pack(">II", 0, n),
                            b"".join(struct.pack(">I", int(s)) for s in sizes)),
                 stss, co)
    minf = O.box(b"minf", O.full_box(b"vmhd", 0, 1, bytes(8)),
                 O.box(b"dinf", O.full_box(b"dref", 0, 0, struct.pack(">I", 1), O.full_box(b"url ", 0, 1))), stbl)
    mdia = O.box(b"mdia", O.full_box(b"mdhd", 0, 0, struct.pack(">IIIIHH", 0, 0, fps_num, dur, 0x55C4, 0)),
                 O.full_box(b"hdlr", 0, 0, bytes(4), b"vide", bytes(12), b"VideoHandler\x00"), minf)
    tkhd = O.full_box(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, 1, 0, dur), bytes(8), struct.pack(">hhHH", 0, 0, 0, 0),
                      O.MATRIX, struct.pack(">II", width << 16, height << 16))
    mvhd = O.full_box(b"mvhd", 0, 0, struct.pack(">IIII", 0, 0, fps_num, dur), struct.pack(">IH", 0x10000, 0x100),
                      bytes(10), O.MATRIX, bytes(24), struct.pack(">I", 2))
    return O.box(b"moov", mvhd, O.box(b"trak", tkhd, mdia))
