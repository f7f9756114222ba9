"""Dense, differentiable float64 model of the rasterizer (TEST INFRASTRUCTURE).

An independent anchor for the oracle's hand-restated backward (SURVEY.md 8c "independent correctness
anchors"): every pixel looks at every splat, order = stable sort by depth, tile membership enters
only as a boolean mask.  Gradients come from torch autograd, so they share no code with
oracle/splat_oracle.c's stage 4/5.  The module's deliberate non-analytic behaviours (Appendix B.4/B.5)
are modelled explicitly:
  - min(0.99, .) passes the gradient straight through;
  - the 1.3*tanfov guard band zeroes d/dt.x (d/dt.y) when clamped and ignores the clamp's t.z dependence;
  - quaternions are used unnormalised, no normalisation Jacobian;
  - dL/dscale is w.r.t. s = mod*scale (no extra `mod` factor) -> model scales as (mod*scale).detach()-shifted;
  - SH colours clamp at 0 with zero gradient where clamped.
Only suitable for small P and images (memory O(H*W*P)).
"""
from __future__ import annotations

import math

import torch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435]


def sh_basis(deg, d):
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    B = [torch.full_like(x, SH_C0)]
    if deg > 0:
        B += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        B += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
    if deg > 2:
        B += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4 * zz - xx - yy),
              SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
              SH_C3[6] * x * (xx - 3 * yy)]
    return torch.stack(B, dim=1)  # (P, nb)


def quat_to_R(q):
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=1).reshape(-1, 3, 3)


# Wrong variants of the chain (`project(..., variant=...)`), each a mistake a per-splat backward could make; the
# per-splat gradient gate of tests/test_oracle_preprocess.py must reject every one of them.
VARIANTS = ("guard_grad", "no_dilation_bwd", "sh3_sign", "colour_clamp_ignored", "normalised_quat", "scale_grad_unmod")


def _value_of(value, grad_path):
    """`value` forward, the derivative of `grad_path` backward."""
    return grad_path + (value - grad_path).detach()


def project(means3D, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, *, shs=None, sh_degree=0,
            colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None, scale_modifier=1.0,
            guard_clamped=None, colour_clamped=None, keep=None, conic_dropped=None, variant=None):
    """The per-splat part of the forward in float64, differentiable: view-space t (P,3), ndc (P,2), pixel centre `pix`
    (P,2), the dilated 2-D covariance `cov2d` (a, b, c) and its determinant, the conic (A, B, C) (P,3), the clamped
    colour `rgb` (P,3) and the depth t.z (P,).

    The float32 side's discrete decisions can be held fixed, as render() does with the tile rectangles:
    `guard_clamped` ((P,2) bool: the guard band clamped t.x / t.y), `colour_clamped` ((P,3) bool: the channel's SH
    sum was below 0) and `keep` ((P,) bool: the splat is rendered; every output of another splat is detached).  Left
    None, each is this model's own.  `conic_dropped` ((P,) bool): the float32 backward's 1 / (det^2 + 1e-7) rounded
    to 0 (det^2 overflows), so no gradient leaves through the conic of those splats (the reference module's guard).
    `variant`: one of VARIANTS (a deliberately wrong backward), or None."""
    dt = torch.float64
    P = means3D.shape[0]
    V = viewmatrix.reshape(16).to(dt)
    Pm = projmatrix.reshape(16).to(dt)
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    x, y, z = means3D[:, 0], means3D[:, 1], means3D[:, 2]
    tx = V[0] * x + V[4] * y + V[8] * z + V[12]
    ty = V[1] * x + V[5] * y + V[9] * z + V[13]
    tz = V[2] * x + V[6] * y + V[10] * z + V[14]
    hx = Pm[0] * x + Pm[4] * y + Pm[8] * z + Pm[12]
    hy = Pm[1] * x + Pm[5] * y + Pm[9] * z + Pm[13]
    hw = Pm[3] * x + Pm[7] * y + Pm[11] * z + Pm[15]
    p_w = 1.0 / (hw + 0.0000001)
    ndc_x, ndc_y = hx * p_w, hy * p_w

    if cov3D_precomp is not None:
        c3 = cov3D_precomp
        Sigma = torch.stack([c3[:, 0], c3[:, 1], c3[:, 2], c3[:, 1], c3[:, 3], c3[:, 4], c3[:, 2], c3[:, 4], c3[:, 5]],
                            dim=1).reshape(P, 3, 3)
    else:
        q = rotations
        if variant == "normalised_quat":
            q = q / q.norm(dim=1, keepdim=True)
        R = quat_to_R(q)
        # gradient w.r.t. s=mod*scale reported as dL/dscale: value mod*scale, derivative 1
        s = scales * scale_modifier if variant == "scale_grad_unmod" else scales + ((scale_modifier - 1.0) * scales).detach()
        Sigma = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)

    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    txtz, tytz = tx / tz, ty / tz
    if guard_clamped is None:
        cx = (txtz < -limx) | (txtz > limx)
        cy = (tytz < -limy) | (tytz > limy)
    else:
        cx, cy = guard_clamped[:, 0], guard_clamped[:, 1]
    if variant == "guard_grad":   # the clamped value, but d/dt.x as if unclamped
        txc = torch.where(cx, _value_of(txtz.clamp(-limx, limx) * tz, tx), tx)
        tyc = torch.where(cy, _value_of(tytz.clamp(-limy, limy) * tz, ty), ty)
    else:
        txc = torch.where(cx, (txtz.clamp(-limx, limx) * tz).detach(), tx)
        tyc = torch.where(cy, (tytz.clamp(-limy, limy) * tz).detach(), ty)
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -(fx * txc) / (tz * tz), zero, fy / tz, -(fy * tyc) / (tz * tz)], dim=1).reshape(P, 2, 3)
    Wv = torch.stack([V[0], V[4], V[8], V[1], V[5], V[9], V[2], V[6], V[10]]).reshape(3, 3)
    T = J @ Wv
    cov = T @ Sigma @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * c - b * b
    # conic with the 1/(det^2+1e-7)-style guard irrelevant at fp64 tolerance
    conA, conB, conC = c / det, -b / det, a / det
    if variant == "no_dilation_bwd":   # the conic's derivatives taken at the undilated covariance
        a0, c0 = cov[:, 0, 0], cov[:, 1, 1]
        det0 = a0 * c0 - b * b
        conA, conB, conC = _value_of(conA, c0 / det0), _value_of(conB, -b / det0), _value_of(conC, a0 / det0)

    if conic_dropped is not None:
        conA, conB, conC = (torch.where(conic_dropped, v.detach(), v) for v in (conA, conB, conC))

    if colors_precomp is not None:
        rgb = colors_precomp
        if colour_clamped is None:
            colour_clamped = torch.zeros_like(rgb, dtype=torch.bool)
    else:
        d = means3D - campos.reshape(1, 3)
        d = d / d.norm(dim=1, keepdim=True)
        B = sh_basis(sh_degree, d)
        if variant == "sh3_sign" and sh_degree > 2:
            B = torch.cat((B[:, :12], -B[:, 12:13], B[:, 13:]), dim=1)
        nb = B.shape[1]
        rgb = (B[:, :, None] * shs[:, :nb, :]).sum(dim=1) + 0.5
        if colour_clamped is None:
            colour_clamped = rgb.detach() < 0
        if variant == "colour_clamp_ignored":
            rgb = _value_of(torch.clamp_min(rgb, 0.0), rgb)
        else:
            rgb = torch.where(colour_clamped, torch.zeros_like(rgb), rgb)

    out = dict(t=torch.stack((tx, ty, tz), 1), ndc=torch.stack((ndc_x, ndc_y), 1),
               pix=torch.stack((((ndc_x + 1.0) * W - 1.0) * 0.5, ((ndc_y + 1.0) * H - 1.0) * 0.5), 1),
               cov2d=torch.stack((a, b, c), 1), det=det, conic=torch.stack((conA, conB, conC), 1), rgb=rgb, depth=tz)
    if keep is not None:
        out = {k: torch.where(keep.reshape((-1,) + (1,) * (v.ndim - 1)), v, v.detach()) for k, v in out.items()}
    out.update(guard_clamped=torch.stack((cx, cy), dim=1), colour_clamped=colour_clamped)
    return out


def render(means3D, means2D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg, *, shs=None,
           sh_degree=0, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None, scale_modifier=1.0,
           radii=None, rect_xy=None, depths=None):
    """All tensor arguments float64.  `radii` (int, from the fp32 oracle) fixes the discrete tile rectangles so the
    comparison is not at the mercy of ceil() knife edges.  `rect_xy` ((P,2) float32 pixel centres, from the fp32
    oracle) also takes the rectangles' centres from there, evaluated in float32 as the oracle does: a centre that
    float32 puts exactly on a truncation edge (an integer pixel centre with (py + r + 15) / 16 integral, say) lands a
    hair below it in float64 and would drop a whole tile row.  `depths` ((P,) float32 view-space depths, from the fp32
    oracle) decides the blend order in place of this model's own depths rounded to float32: two splats a rounding
    apart in depth composite in the oracle's order.  Returns (image (3,H,W), aux dict); aux also holds the discrete
    decisions (`keep`, `alpha_clamped`, `colour_clamped`, `guard_clamped`) a caller can hold fixed."""
    dt = torch.float64
    pr = project(means3D, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, shs=shs, sh_degree=sh_degree,
                 colors_precomp=colors_precomp, scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp,
                 scale_modifier=scale_modifier)
    tz = pr["depth"]
    in_front = tz > 0.2
    a, c, det = pr["cov2d"][:, 0], pr["cov2d"][:, 2], pr["det"]
    conA, conB, conC = pr["conic"].unbind(1)
    px = pr["pix"][:, 0] + means2D[:, 0] * (0.5 * W)
    py = pr["pix"][:, 1] + means2D[:, 1] * (0.5 * H)
    rgb, colour_clamped = pr["rgb"], pr["colour_clamped"]
    cx, cy = pr["guard_clamped"].unbind(1)

    # discrete tile rectangles
    gx, gy = (W + 15) // 16, (H + 15) // 16
    if radii is None:
        mid = 0.5 * (a + c)
        lam = mid + torch.sqrt(torch.clamp_min(mid * mid - det, 0.1))
        radii = torch.ceil(3.0 * torch.sqrt(lam)).to(torch.int64)
    if rect_xy is None:
        rad = radii.to(dt)
        pxd, pyd = px.detach(), py.detach()
    else:  # splat_oracle.c tile_rect, float32 throughout
        rad = radii.to(torch.float32)
        pxd, pyd = rect_xy[:, 0].to(torch.float32), rect_xy[:, 1].to(torch.float32)
    x0 = torch.clamp(((pxd - rad) / 16).trunc(), 0, gx).to(dt)
    y0 = torch.clamp(((pyd - rad) / 16).trunc(), 0, gy).to(dt)
    x1 = torch.clamp(((pxd + rad + 15) / 16).trunc(), 0, gx).to(dt)
    y1 = torch.clamp(((pyd + rad + 15) / 16).trunc(), 0, gy).to(dt)
    visible = in_front & (radii > 0) & ((x1 - x0) * (y1 - y0) > 0)

    key = tz.detach() if depths is None else depths
    order = torch.argsort(key.to(torch.float32), stable=True)  # fp32 depth bits decide, ties by id
    ys, xs = torch.meshgrid(torch.arange(H, dtype=dt), torch.arange(W, dtype=dt), indexing="ij")
    pixx, pixy = xs.reshape(-1, 1), ys.reshape(-1, 1)  # (HW,1)
    tilex, tiley = (pixx / 16).floor(), (pixy / 16).floor()

    def g(v):
        return v[order][None, :]

    member = g(visible) & (tilex >= g(x0)) & (tilex < g(x1)) & (tiley >= g(y0)) & (tiley < g(y1))
    dx, dy = g(px) - pixx, g(py) - pixy
    power = -0.5 * (g(conA) * dx * dx + g(conC) * dy * dy) - g(conB) * dx * dy
    Gs = torch.exp(torch.clamp_max(power, 0.0))
    og = g(opacities.reshape(-1)) * Gs
    alpha = og + (torch.clamp_max(og, 0.99) - og).detach()
    valid = member & (power <= 0) & (alpha.detach() >= 1.0 / 255.0)
    aeff = torch.where(valid, alpha, torch.zeros_like(alpha))
    one_minus = 1.0 - aeff
    T_incl = torch.cumprod(one_minus, dim=1)
    T_before = torch.cat((torch.ones_like(T_incl[:, :1]), T_incl[:, :-1]), dim=1)
    stop = valid & (T_incl.detach() < 0.0001)
    stopped = torch.cumsum(stop.to(torch.int64), dim=1) > 0  # inclusive: the stopping instance itself is dropped
    keep = valid & ~stopped
    w = torch.where(keep, aeff * T_before, torch.zeros_like(aeff))
    C = w @ rgb[order]  # (HW,3)
    T_final = torch.where(keep, one_minus, torch.ones_like(one_minus)).prod(dim=1)
    out = C + T_final[:, None] * bg.reshape(1, 3)
    img = out.t().reshape(3, H, W)
    return img, dict(radii=radii, visible=visible, T_final=T_final.reshape(H, W), n_keep=keep.sum(dim=1).reshape(H, W),
                     keep=keep, alpha_clamped=og.detach() > 0.99, colour_clamped=colour_clamped,
                     guard_clamped=torch.stack((cx, cy), dim=1))
