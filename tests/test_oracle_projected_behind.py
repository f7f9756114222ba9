"""CPU: the backward blend's dL/dalpha in the form it carries behind each pixel -- one dL/dpixel-weighted sum

    U_i = sum_{j>i} (c_j . d) alpha_j T_j + T_final (bg . d),   dL/dalpha_i = T_i (c_i . d) - U_i / (1 - alpha_i)

(blend.cu visit_bands) -- is no further from float64 than the reference's form, which carries the colour composited
behind the splat per channel and takes T_i ((c_i - behind) . d) - T_final (bg . d) / (1 - alpha_i).

One pixel's reverse walk is restated in float32 numpy in both forms, over every pixel of the walk scenes and the
adversarial scenes, from the oracle's forward state (alphas, final_T, n_contrib), with and without the depth plane
(a fourth channel: colour z, background 0, dL/dalpha folded into the background term).  Both are measured against
the same walk in float64, as the largest error over the largest float64 value of each tensor: the per-pair dL/dalpha
and the per-splat dL/dopacity (sum over pixels of G dL/dalpha).  The saturating stacks (T down to 1e-4) are where a
cancellation of the unnormalised sum would show.

Both forms stay within REL_BOUND, a few float32 roundings of each tensor's largest value.  The projected form's error
is not smaller than the channel form's: on these scenes it is 0.7x to 2.3x of it, 8e-7 at most (DESIGN.md section 5
has the table); a cancellation would show as orders of magnitude more."""
import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import helpers as h
from tests import walk_scenes as WS

F32, F64 = np.float32, np.float64
SCENES = [("walk", n) for n in WS.WALK] + [("adversarial", n) for n in A.BUILDERS]
REL_BOUND = 2.0 ** -20


def _fma(a, b, c):
    """fmaf in float32: the product is exact in float64, the sum rounds (a double rounding may move the last ulp)."""
    return (F64(1) * a * b + c).astype(F32)


def _walk(st, bg, d, dD, dA, form):
    """dL/dalpha of every (stream position, pixel) pair the blend took, zero elsewhere, walked in reverse as the
    backward blend walks it: form "channels" (the reference's), "projected" (U) or "float64" (channels, in float64).
    Returns (pair values [N, H*W], G [N, H*W])."""
    W, H, gx = st.W, st.H, (st.W + 15) // 16
    da = dD is not None
    ft = F64 if form == "float64" else F32
    out = np.zeros((st.N, W * H), F64)
    Gs = np.zeros((st.N, W * H), F64)
    ly, lx = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
    for tile in range(st.ranges.shape[0]):
        r0, r1 = int(st.ranges[tile, 0]), int(st.ranges[tile, 1])
        if r1 <= r0:
            continue
        xs, ys = (tile % gx) * 16 + lx.reshape(-1), (tile // gx) * 16 + ly.reshape(-1)
        inside = (xs < W) & (ys < H)
        pix = ys[inside] * W + xs[inside]
        ids = st.vals_sorted[r0:r1].astype(np.int64)
        co = st.conic_opacity[ids]
        dx = st.xy[ids, 0][:, None] - xs[inside][None, :].astype(F32)
        dy = st.xy[ids, 1][:, None] - ys[inside][None, :].astype(F32)
        power = F32(-0.5) * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
        G = np.exp(np.minimum(power, F32(0)))
        alpha = np.minimum(F32(0.99), co[:, 3:4] * G)
        live = np.arange(r1 - r0)[:, None] < st.n_contrib.reshape(-1)[pix][None, :].astype(np.int64)
        valid = live & (power <= 0) & (alpha >= A.ALPHA_MIN)
        dp = [ft(d[c].reshape(-1)[pix]) for c in range(3)] + ([ft(dD.reshape(-1)[pix])] if da else [])
        T = ft(st.final_T.reshape(-1)[pix])
        bgd = ft(bg[0]) * dp[0] + ft(bg[1]) * dp[1] + ft(bg[2]) * dp[2]
        bgT = T * ((bgd - ft(dA.reshape(-1)[pix])) if da else bgd)
        behind = [np.zeros_like(T) for _ in dp]
        U = bgT
        for k in range(r1 - r0 - 1, -1, -1):
            v = valid[k]
            al = np.where(v, alpha[k], F32(0)).astype(ft)
            ra = np.where(v, ft(1) / (ft(1) - ft(alpha[k])), ft(1)).astype(ft)
            Tn = T * ra
            T = Tn
            c = [ft(st.rgb[ids[k], ch]) for ch in range(3)] + ([ft(st.depths[ids[k]])] if da else [])
            if form == "projected":
                cd = c[0] * dp[0]
                for ch in range(1, len(dp)):
                    cd = _fma(c[ch], dp[ch], cd)
                dLda = _fma(Tn, cd, -(U * ra))
                U = _fma(al * Tn, cd, U)
            else:
                e = [c[ch] - behind[ch] for ch in range(len(dp))]
                dLda = e[0] * dp[0]
                for ch in range(1, len(dp)):
                    dLda = dLda + e[ch] * dp[ch] if form == "float64" else _fma(e[ch], dp[ch], dLda)
                if form == "float64":
                    dLda = dLda * Tn - bgT * ra
                    behind = [behind[ch] + al * e[ch] for ch in range(len(dp))]
                else:
                    dLda = _fma(dLda, Tn, -(bgT * ra))
                    behind = [_fma(al, e[ch], behind[ch]) for ch in range(len(dp))]
            out[r0 + k, pix] = np.where(v, dLda, 0)
            Gs[r0 + k, pix] = np.where(v, G[k], 0)
    return out, Gs


def _state(kind, name):
    sc = WS.build(name) if kind == "walk" else A.build(name)
    return sc, h.oracle_forward(sc)


def _rel(x, ref):
    return float(np.abs(x - ref).max() / max(np.abs(ref).max(), 1e-30))


@pytest.mark.parametrize("da", [False, True], ids=["rgb", "depth_alpha"])
@pytest.mark.parametrize("kind,name", SCENES)
def test_projected_sum_is_no_further_from_float64(kind, name, da):
    sc, st = _state(kind, name)
    g = torch.Generator().manual_seed(7)
    d = torch.randn(3, st.H, st.W, generator=g).numpy()
    dD = torch.randn(st.H, st.W, generator=g).numpy() if da else None
    dA = torch.randn(st.H, st.W, generator=g).numpy() if da else None
    bg = sc["bg"].numpy()
    ref, G = _walk(st, bg, d, dD, dA, "float64")
    assert np.count_nonzero(ref) > 0
    ids = st.vals_sorted[:st.N].astype(np.int64)
    err = {}
    for form in ("channels", "projected"):
        x, _ = _walk(st, bg, d, dD, dA, form)
        op = np.zeros(st.P)
        np.add.at(op, ids, (G * x).sum(axis=1))
        op64 = np.zeros(st.P)
        np.add.at(op64, ids, (G * ref).sum(axis=1))
        err[form] = (_rel(x, ref), _rel(op, op64))
    print(f"[projected] {name} {'DA' if da else 'rgb'}: dL/dalpha rel err channels {err['channels'][0]:.2e} "
          f"projected {err['projected'][0]:.2e}; dL/dopacity channels {err['channels'][1]:.2e} "
          f"projected {err['projected'][1]:.2e}")
    for i, what in enumerate(("dL/dalpha", "dL/dopacity")):
        for form in ("channels", "projected"):
            assert err[form][i] <= REL_BOUND, f"{name}: {what} of the {form} form {err[form][i]:.2e} from float64"
