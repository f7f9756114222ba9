"""A plain restatement of the device H.264 encode with I_NxN macroblocks (csrc/h264.cu gab200_h264_encode_flags with
GAB200_H264_INTRA4X4), written from ITU-T H.264 clauses 7.3.5.1, 8.3.1 and 9.2 on top of oracle/h264.py,
tests/h264_stream_oracle.py and tests/h264_deblock_oracle.py, which it reuses unchanged -- what
tests/test_gpu_video_intra4x4.py compares the device's bytes with, and what FFmpeg's decoder referees in
tests/test_oracle_h264_intra4x4.py.

    frames = encode_stream(rgbs, qp, gop, deblock=False)  # [dict(sample, recon, filtered, types, mvs, report), ...]
    data = mp4([f["sample"] for f in frames], W, H, qp, gop=gop)

The stream is tests/h264_stream_oracle.py's (tests/h264_deblock_oracle.py's when deblocked) with one more intra
candidate.  Each macroblock also codes its 16 luma 4x4 blocks in decode order (luma4x4BlkIdx): a block takes, among
the Intra_4x4 modes whose samples are available (8.3.1.2), the one of least SATD(src - pred) + lambda * (1 when it
is predIntra4x4PredMode, else 4), ties to the lower mode; block 5 never takes modes 3 or 7 (they read the macroblock
above right); its 16 coefficients are quantised with the intra dead zone and reconstructed before the next block
predicts.  I_NxN replaces I_16x16 when the blocks' costs + I4_BIAS * lambda sum below I_16x16's least luma SATD; in a
P picture the cheaper candidate meets the inter cost through INTRA_BIAS.  I_PCM replaces I_NxN as it replaces
I_16x16.  Each diagonal's macroblocks are coded at once in numpy, block by block.
"""
from __future__ import annotations

import struct

import numpy as np

from oracle import h264 as O
from tests import h264_deblock_oracle as D
from tests import h264_stream_oracle as S

I4_BIAS = 8                      # I_NxN's handicap against I_16x16, in units of lambda
# Table 9-4, intra column: coded_block_pattern -> codeNum
INTRA_CBP_CODE = [0] * 48
for _k, _c in enumerate([47, 31, 15, 0, 23, 27, 29, 30, 7, 11, 13, 14, 39, 43, 45, 46, 16, 3, 5, 10, 12, 19, 21, 26,
                         28, 35, 37, 42, 44, 1, 2, 4, 8, 17, 18, 20, 24, 6, 9, 22, 25, 32, 33, 34, 36, 40, 38, 41]):
    INTRA_CBP_CODE[_c] = _k
MODE_NAMES = ("V", "H", "DC", "DDL", "DDR", "VR", "HD", "VL", "HU")


def blk_idx(bx: int, by: int) -> int:
    return 8 * (by >> 1) + 4 * (bx >> 1) + 2 * (by & 1) + (bx & 1)


# ---- Intra_4x4 prediction (8.3.1.2) as weights over the edge e: e[3 - j] = p[-1, j], e[4] = p[-1, -1],
# e[5 + i] = p[i, -1] (i = 0 .. 7) --------------------------------------------------------------------------------------
def _e(i, j):
    return 5 + i if j < 0 else 3 - j


def _taps(mode, x, y):
    """[(edge index, weight)] of mode's sample (x, y); the weights sum to 1, 2 or 4 (the shift)."""
    P = _e

    def f3(a, b, c):
        return [(a, 1), (b, 2), (c, 1)]

    def f2(a, b):
        return [(a, 1), (b, 1)]

    if mode == 0:
        return [(P(x, -1), 1)]
    if mode == 1:
        return [(P(-1, y), 1)]
    if mode == 3:
        if x == 3 and y == 3:
            return [(P(6, -1), 1), (P(7, -1), 3)]
        return f3(P(x + y, -1), P(x + y + 1, -1), P(x + y + 2, -1))
    if mode == 4:
        if x > y:
            return f3(P(x - y - 2, -1), P(x - y - 1, -1), P(x - y, -1))
        if x < y:
            return f3(P(-1, y - x - 2), P(-1, y - x - 1), P(-1, y - x))
        return f3(P(0, -1), P(-1, -1), P(-1, 0))
    if mode == 5:
        z = 2 * x - y
        if z >= 0 and z % 2 == 0:
            return f2(P(x - (y >> 1) - 1, -1), P(x - (y >> 1), -1))
        if z > 0:
            return f3(P(x - (y >> 1) - 2, -1), P(x - (y >> 1) - 1, -1), P(x - (y >> 1), -1))
        if z == -1:
            return f3(P(-1, 0), P(-1, -1), P(0, -1))
        return f3(P(-1, y - 1), P(-1, y - 2), P(-1, y - 3))
    if mode == 6:
        z = 2 * y - x
        if z >= 0 and z % 2 == 0:
            return f2(P(-1, y - (x >> 1) - 1), P(-1, y - (x >> 1)))
        if z > 0:
            return f3(P(-1, y - (x >> 1) - 2), P(-1, y - (x >> 1) - 1), P(-1, y - (x >> 1)))
        if z == -1:
            return f3(P(-1, 0), P(-1, -1), P(0, -1))
        return f3(P(x - 1, -1), P(x - 2, -1), P(x - 3, -1))
    if mode == 7:
        if y % 2 == 0:
            return f2(P(x + (y >> 1), -1), P(x + (y >> 1) + 1, -1))
        return f3(P(x + (y >> 1), -1), P(x + (y >> 1) + 1, -1), P(x + (y >> 1) + 2, -1))
    z = x + 2 * y                                        # mode 8
    if z > 5:
        return [(P(-1, 3), 1)]
    if z == 5:
        return [(P(-1, 2), 1), (P(-1, 3), 3)]
    if z % 2 == 0:
        return f2(P(-1, y + (x >> 1)), P(-1, y + (x >> 1) + 1))
    return f3(P(-1, y + (x >> 1)), P(-1, y + (x >> 1) + 1), P(-1, y + (x >> 1) + 2))


W4 = np.zeros((9, 16, 13), np.int64)
SH4 = np.zeros((9, 16), np.int64)
for _m in range(9):
    if _m == 2:
        continue
    for _y in range(4):
        for _x in range(4):
            for _i, _w in _taps(_m, _x, _y):
                W4[_m, 4 * _y + _x, _i] += _w
            SH4[_m, 4 * _y + _x] = int(W4[_m, 4 * _y + _x].sum()).bit_length() - 1


def predict4(e, al, at):
    """(M, 9, 16) predictions (raster) of the nine modes from edges e (M, 13) with p[4..7, -1] substituted where
    absent; al / at (M,): left / top available (mode 2's DC)."""
    e = np.asarray(e, np.int64)
    p = (np.einsum("mi,kpi->mkp", e, W4) + ((1 << SH4) >> 1)) >> SH4
    sl, st = e[:, 0:4].sum(1), e[:, 5:9].sum(1)
    dc = np.where(al & at, (sl + st + 4) >> 3, np.where(at, (st + 2) >> 2, np.where(al, (sl + 2) >> 2, 128)))
    p[:, 2] = dc[:, None]
    return p


def available4(bx, by, al, at):
    """(M, 9) the modes a block may take: 8.3.1.2's availability, and never 3 or 7 in block 5."""
    both = al & at
    ok = np.stack([at, al, np.ones_like(al), at, both, both, both, at, al], 1)
    if (bx, by) == (3, 0):
        ok[:, [3, 7]] = False
    return ok


# ---- the macroblock's I_NxN candidate ----------------------------------------------------------------------------
def code_i4(src, top, left, tl, has_t, has_l, mx, my, qp, nxn_grid, mode_grid):
    """The I_NxN candidate of M macroblocks: src (M, 16, 16), their reconstructed top / left (M, 16), tl (M,),
    neighbours' I_NxN flags and modes (hm, wm) / (hm, wm, 4, 4).  Returns dict(cost (M,), modes, pm (M, 4, 4)
    [by, bx], lev (M, 4, 4, 4, 4) [by, bx, y, x], rec (M, 16, 16), tr_sub (M, 4, 4) bool)."""
    M = src.shape[0]
    L = S.lam(qp)
    loc = np.zeros((M, 17, 17), np.int64)             # loc[y + 1, x + 1] = p[x, y] of the macroblock
    loc[:, 0, 0] = tl
    loc[:, 0, 1:] = top
    loc[:, 1:, 0] = left
    modes = np.zeros((M, 4, 4), np.int64)
    pms = np.zeros((M, 4, 4), np.int64)
    lev = np.zeros((M, 4, 4, 4, 4), np.int64)
    sub = np.zeros((M, 4, 4), bool)
    cost = np.zeros(M, np.int64)
    for k, (bx, by) in enumerate(O.LUMA_BLK):
        al = np.full(M, bx > 0) | has_l
        at = np.full(M, by > 0) | has_t
        atr = np.full(M, False) if bx == 3 else (has_t.copy() if by == 0 else np.full(M, blk_idx(bx + 1, by - 1) < k))
        x0, y0 = 4 * bx, 4 * by
        e = np.zeros((M, 13), np.int64)
        for j in range(4):
            e[:, 3 - j] = loc[:, y0 + 1 + j, x0]
        e[:, 4] = loc[:, y0, x0]
        for i in range(8):
            far = loc[:, y0, min(x0 + 1 + i, 16)]
            e[:, 5 + i] = loc[:, y0, x0 + 1 + i] if i < 4 else np.where(atr, far, loc[:, y0, x0 + 4])
        e[:, 0:4] *= al[:, None]
        e[:, 5:13] *= at[:, None]
        e[:, 4] *= al & at
        pred = predict4(e, al, at)
        blk = src[:, y0:y0 + 4, x0:x0 + 4].reshape(M, 1, 16)
        satd = O.satd((blk - pred).reshape(M, 9, 4, 4))
        # predIntra4x4PredMode (8.3.1.1)
        if bx > 0:
            a = modes[:, by, bx - 1]
        else:
            xl = np.maximum(mx - 1, 0)
            a = np.where(nxn_grid[my, xl], mode_grid[my, xl, by, 3], 2)
        if by > 0:
            b = modes[:, by - 1, bx]
        else:
            yt = np.maximum(my - 1, 0)
            b = np.where(nxn_grid[yt, mx], mode_grid[yt, mx, 3, bx], 2)
        pm = np.where(al & at, np.minimum(a, b), 2)
        c = satd + L * np.where(np.arange(9)[None, :] == pm[:, None], 1, 4)
        c = np.where(available4(bx, by, al, at), c, np.iinfo(np.int64).max)
        m = np.argmin(c, 1)
        cost += c[np.arange(M), m]
        p = pred[np.arange(M), m].reshape(M, 4, 4)
        w = O.CF @ (blk.reshape(M, 4, 4) - p) @ O.CF.T
        lv = O.quant(w, qp, O.MF[qp % 6][O.POS], False)
        rec = np.clip(p + O.idct4(O.dequant_ac(lv, qp)), 0, 255)
        loc[:, y0 + 1:y0 + 5, x0 + 1:x0 + 5] = rec
        modes[:, by, bx], pms[:, by, bx], lev[:, by, bx] = m, pm, lv
        sub[:, by, bx] = at & ~atr & np.isin(m, (3, 7))
    return dict(cost=cost, modes=modes, pm=pms, lev=lev, rec=loc[:, 1:, 1:], tr_sub=sub)


def i4_bits(mx, my, is_p, modes, pm, cmode, lev, cdcl, cacl, tl_, tc_, report):
    """The I_NxN macroblock_layer's bits; fills its totals into the grids."""
    cbpl = 0
    for k in range(4):
        if np.any(lev[2 * (k // 2):2 * (k // 2) + 2, 2 * (k % 2):2 * (k % 2) + 2]):
            cbpl |= 1 << k
    cbpc = 2 if np.any(cacl) else 1 if np.any(cdcl) else 0
    for bx, by in O.LUMA_BLK:
        tl_[4 * my + by, 4 * mx + bx] = np.count_nonzero(lev[by, bx])
    for c in range(2):
        for by in range(2):
            for bx in range(2):
                tc_[c][2 * my + by, 2 * mx + bx] = np.count_nonzero(cacl[c, by, bx]) if cbpc == 2 else 0
    b = O.Bits()
    b.ue(5 if is_p else 0)
    for bx, by in O.LUMA_BLK:
        m, p = int(modes[by, bx]), int(pm[by, bx])
        if m == p:
            b.u(1, 1)
            report.add(("prev_intra4x4_pred_mode_flag", 1))
        else:
            r = m if m < p else m - 1
            b.u(0, 1)
            b.u(r, 3)
            report.add(("prev_intra4x4_pred_mode_flag", 0))
            report.add(("rem_intra4x4_pred_mode", r))
    b.ue(cmode)
    cbp = cbpl | cbpc << 4
    b.ue(INTRA_CBP_CODE[cbp])
    report.add(("intra_cbp_luma", cbpl))
    report.add(("intra_cbp_chroma", cbpc))
    if cbp:
        b.se(0)
    for bx, by in O.LUMA_BLK:
        if (cbpl >> ((by // 2) * 2 + bx // 2)) & 1:
            O.residual_block(b, lev[by, bx].reshape(16)[O.ZIGZAG], O.nc_of(tl_, 4 * mx + bx, 4 * my + by), report)
    if cbpc:
        for c in range(2):
            O.residual_block(b, cdcl[c].reshape(4), -1, report)
    if cbpc == 2:
        for c in range(2):
            for by in range(2):
                for bx in range(2):
                    O.residual_block(b, cacl[c, by, bx].reshape(16)[O.ZIGZAG[1:]],
                                     O.nc_of(tc_[c], 2 * mx + bx, 2 * my + by), report)
    return b


# ---- the encode ----------------------------------------------------------------------------------------------------
def encode_picture(rgb, qp, ref, frame_num):
    """One picture: an IDR picture when ref is None, else a P picture referring to the padded picture ref.  Returns
    dict(sample, recon (padded), types (hm, wm) 'I', 'I4', 'PCM', 'P' or 'P_Skip', mvs, modes (hm, wm, 4, 4),
    totals (4 hm, 4 wm), report)."""
    rgb = np.asarray(rgb, np.uint8)
    H, W, _ = rgb.shape
    qpc = O.CHROMA_QP[qp]
    ys, cbs, crs = O.rgb_to_yuv(rgb)
    hc, wc = ys.shape
    hm, wm = hc // 16, wc // 16
    is_p = ref is not None
    report = set()
    if not is_p:
        mv, ipred = np.zeros((hm, wm, 2), np.int64), np.zeros((hm, wm, 16, 16), np.int64)
        icost = np.full((hm, wm), np.iinfo(np.int64).max // 2)
        cpred = [np.zeros((hm, wm, 8, 8), np.int64)] * 2
    else:
        mv, ipred, icost = S.search(ys, ref[0], qp)
        X, Y = S._mb_grid(hm, wm, 8)
        cpred = [S.chroma_pred(r, X, Y, mv[..., 0, None, None], mv[..., 1, None, None]) for r in ref[1:]]
    L = S.lam(qp)
    ry, rcb, rcr = np.zeros_like(ys), np.zeros_like(cbs), np.zeros_like(crs)
    tl_ = np.zeros((4 * hm, 4 * wm), np.int64)
    tc_ = [np.zeros((2 * hm, 2 * wm), np.int64) for _ in range(2)]
    types = np.full((hm, wm), "P", dtype=object)
    cbps = np.zeros((hm, wm), np.int64)
    nxn_grid = np.zeros((hm, wm), bool)
    mode_grid = np.zeros((hm, wm, 4, 4), np.int64)
    mbbits = {}
    i4_info = []                                       # (x, y, tr_sub, modes) of the I_NxN macroblocks
    for d in range(wm + hm - 1):
        mx = np.arange(max(0, d - hm + 1), min(d, wm - 1) + 1)
        my = d - mx
        has_l, has_t = mx > 0, my > 0
        M = len(mx)
        yy = (16 * my)[:, None] + np.arange(16)
        xx = (16 * mx)[:, None] + np.arange(16)
        src = ys[yy[:, :, None], xx[:, None, :]].astype(np.int64)
        top = np.where(has_t[:, None], ry[np.maximum(16 * my - 1, 0)[:, None], xx], 0)
        left = np.where(has_l[:, None], ry[yy, np.maximum(16 * mx - 1, 0)[:, None]], 0)
        tlv = np.where(has_t & has_l, ry[np.maximum(16 * my - 1, 0), np.maximum(16 * mx - 1, 0)], 0)
        pl = O.predict(top, left, tlv, has_t, has_l, 16, False)
        lav = np.stack([has_t, has_l, np.ones(M, bool), has_t & has_l], 1)
        lcost = np.where(lav, O.satd(src[:, None] - pl), np.iinfo(np.int64).max)
        lm = np.argmin(lcost, 1)
        i4 = code_i4(src, top, left, tlv, has_t, has_l, mx, my, qp, nxn_grid, mode_grid)
        i16 = lcost[np.arange(M), lm]
        nxn = i4["cost"] + I4_BIAS * L < i16
        intra = np.where(nxn, i4["cost"] + I4_BIAS * L, i16) + S.INTRA_BIAS * L < icost[my, mx]
        cy = (8 * my)[:, None] + np.arange(8)
        cx = (8 * mx)[:, None] + np.arange(8)
        csrc, cpa = [], []
        for plane, rp in ((cbs, rcb), (crs, rcr)):
            csrc.append(plane[cy[:, :, None], cx[:, None, :]])
            t = np.where(has_t[:, None], rp[np.maximum(8 * my - 1, 0)[:, None], cx], 0)
            lf = np.where(has_l[:, None], rp[cy, np.maximum(8 * mx - 1, 0)[:, None]], 0)
            tv = np.where(has_t & has_l, rp[np.maximum(8 * my - 1, 0), np.maximum(8 * mx - 1, 0)], 0)
            cpa.append(O.predict(t, lf, tv, has_t, has_l, 8, True))
        cav = np.stack([np.ones(M, bool), has_l, has_t, has_t & has_l], 1)
        cm = O.choose(cpa, csrc, cav)
        lp = pl[np.arange(M), lm]
        dcl, acl, rres = O.code_luma(src - lp, qp)
        ires = [O.code_chroma(s - p[np.arange(M), cm], qpc) for s, p in zip(csrc, cpa)]
        ip = ipred[my, mx]
        lev, pres = S.code_luma_inter(src - ip, qp)
        cp = [c[my, mx] for c in cpred]
        pres_c = [S.code_chroma_inter(s - p, qpc) for s, p in zip(csrc, cp)]
        for i in range(M):
            x, y = int(mx[i]), int(my[i])
            b = None
            if intra[i]:
                cdcl = np.stack([r[0][i] for r in ires])
                cacl = np.stack([r[1][i] for r in ires])
                rep = set()
                if nxn[i]:
                    over = max(np.abs(i4["lev"][i]).max(), np.abs(cdcl).max(), np.abs(cacl).max())
                    if over <= O.MAX_LEVEL:
                        b = i4_bits(x, y, is_p, i4["modes"][i], i4["pm"][i], int(cm[i]), i4["lev"][i], cdcl, cacl,
                                    tl_, tc_, rep)
                        lrec = i4["rec"][i]
                        kind = "I4"
                else:
                    over = max(np.abs(dcl[i]).max(), np.abs(acl[i]).max(), np.abs(cdcl).max(), np.abs(cacl).max())
                    if over <= O.MAX_LEVEL:
                        b = S.intra_bits(x, y, int(lm[i]), int(cm[i]), dcl[i], acl[i], cdcl, cacl, tl_, tc_, rep,
                                         5 if is_p else 0)
                        lrec = np.clip(lp[i] + rres[i], 0, 255)
                        kind = "I"
                if b is not None and b.n <= O.PCM_BITS:
                    report |= rep
                    types[y, x] = kind
                    report.add(("mb", "I_NxN" if kind == "I4" else "I_16x16"))
                    if kind == "I4":
                        nxn_grid[y, x] = True
                        mode_grid[y, x] = i4["modes"][i]
                        i4_info.append((x, y, i4["tr_sub"][i], i4["modes"][i]))
                    ry[16 * y:16 * y + 16, 16 * x:16 * x + 16] = lrec
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
                    rb, cbp = S.inter_residual_bits(x, y, lev[i], cdcl, cacl, tl_, tc_, rep)
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
    mvs = np.where((types == "P")[..., None], mv, 0)
    if is_p:
        mvp, mvps = S.predictors(types, mvs)
        skipped = (types == "P") & (cbps == 0) & np.all(mvs == mvps, -1)
    else:
        skipped = np.zeros((hm, wm), bool)
    b = O.Bits()
    if is_p:
        S.p_slice_header(b, frame_num)
    else:
        O.slice_header(b)
    parts, n, run = [b.bits()], b.n, 0
    for y in range(hm):
        for x in range(wm):
            if skipped[y, x]:
                run += 1
                continue
            r = O.Bits()
            if is_p:
                r.ue(run)
            run = 0
            if types[y, x] == "PCM":
                if is_p:
                    s = r.bits() + S._pcm_bits(n + r.n, ys, cbs, crs, x, y)
                else:
                    head = "000011010" + "0" * (-(n + 9) % 8)
                    smp = np.concatenate([ys[16 * y:16 * y + 16, 16 * x:16 * x + 16].ravel(),
                                          cbs[8 * y:8 * y + 8, 8 * x:8 * x + 8].ravel(),
                                          crs[8 * y:8 * y + 8, 8 * x:8 * x + 8].ravel()])
                    s = head + "".join(format(int(v), "08b") for v in smp)
            elif types[y, x] in ("I", "I4"):
                s = r.bits() + mbbits[(y, x)]
            else:
                m = O.Bits()
                m.ue(0)
                dv = mvs[y, x] - mvp[y, x]
                m.se(int(dv[0]))
                m.se(int(dv[1]))
                s = r.bits() + m.bits() + mbbits[(y, x)]
            parts.append(s)
            n += len(s)
    if run:
        r = O.Bits()
        r.ue(run)
        parts.append(r.bits())
    parts.append("1")
    esc, _ = O.emulation_prevention(O.to_bytes("".join(parts)))
    body = (b"\x61" if is_p else b"\x65") + esc
    sample = struct.pack(">I", len(body)) + body
    assert len(sample) <= (S.p_bound(W, H) if is_p else O.bound(W, H))
    t = np.where(skipped, "P_Skip", types)
    _report_i4(report, t, i4_info, wm, is_p)
    return dict(sample=sample, recon=(ry, rcb, rcr), types=t, mvs=mvs, modes=mode_grid, totals=tl_, report=report)


def _report_i4(report, types, i4_info, wm, is_p):
    """The corpus paths of the picture's I_NxN macroblocks (tests/test_oracle_h264_intra4x4.py asserts them)."""
    hm = types.shape[0]
    names = {"I": "I_16x16", "I4": "I_NxN", "PCM": "I_PCM", "P": "P_L0_16x16", "P_Skip": "P_Skip"}
    for x, y, sub, modes in i4_info:
        if is_p:
            report.add(("i4_in_p",))
        for nx, ny in ((x - 1, y), (x, y - 1)):
            report.add(("i4_neighbour", names[types[ny, nx]] if nx >= 0 and ny >= 0 else "unavailable"))
        for m in np.unique(modes):
            report.add(("i4_mode", int(m)))
        for side, at in (("top", y == 0), ("left", x == 0), ("right", x == wm - 1)):
            if at:
                for m in np.unique(modes):
                    report.add(("i4_mode_at", side, int(m)))
        if sub.any():
            report.add(("i4_top_right_substituted",))
        report.add(("i4_block5", "with_C" if y > 0 and x < wm - 1 else "without_C"))


def encode_stream(frames, qp: int, gop: int, deblock: bool = False, start: int = 0, ref=None) -> list:
    """Per frame dict(sample, recon (padded, unfiltered), filtered (padded, the decoder's output), types, mvs, modes,
    report).  start: the stream position of frames[0]; ref: the (filtered) padded picture before it (when start %
    gop)."""
    if not 1 <= gop <= 65535:
        raise ValueError(f"gop must be in 1..65535, got {gop}")
    out = []
    for k, rgb in enumerate(frames):
        n = start + k
        f = encode_picture(rgb, qp, None if n % gop == 0 else ref, (n % gop) % 16)
        if deblock:
            types = np.where(f["types"] == "I4", "I", f["types"])
            f["filtered"], f["paths"] = D.deblock(f["recon"], types, f["mvs"], f["totals"], qp, n % gop != 0)
            f["sample"] = D.deblocked_sample(f["sample"])
        else:
            f["filtered"] = f["recon"]
        ref = f["filtered"]
        out.append(f)
    return out


crop = S.crop
# the parameter sets and the container are the same with and without I_NxN
mp4 = S.mp4
