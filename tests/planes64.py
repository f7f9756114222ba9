"""The alpha and depth planes in float64 (TEST INFRASTRUCTURE), composed from oracle/dense64.py without changing it.

dense64.render returns the differentiable T_final of its walk, and its image is linear in the colours with the walk
independent of them, so
    alpha = 1 - T_final                                  (aux["T_final"] of the colour render)
    depth = image[0] of the same render with colours (z, 0, 0) and background 0, z = V[2] x + V[6] y + V[10] z + V[14]
are the planes of include/gab200_rasterizer.h, differentiable in every input by float64 autograd, with no code shared
with the library or the C oracle.  The C-oracle side is the same identity in float32: alpha = 1 - final_T, depth =
out_color[0] of an oracle forward with colours (depths, 0, 0) and background 0."""
from __future__ import annotations

import numpy as np
import torch

from oracle import dense64
from oracle import rasterizer as orc


def view_depth(means3D, viewmatrix):
    V = viewmatrix.reshape(16).to(means3D.dtype)
    return V[2] * means3D[:, 0] + V[6] * means3D[:, 1] + V[10] * means3D[:, 2] + V[14]


def render(means3D, means2D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg, **kw):
    """dense64.render's arguments (float64) -> (image (3,H,W), alpha (1,H,W), depth (1,H,W), aux)."""
    img, aux = dense64.render(means3D, means2D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg,
                              **kw)
    z = view_depth(means3D, viewmatrix)
    zc = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], dim=1)
    kz = {k: v for k, v in kw.items() if k not in ("shs", "sh_degree", "colors_precomp")}
    img_z, _ = dense64.render(means3D, means2D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy,
                              torch.zeros_like(bg), colors_precomp=zc, **kz)
    return img, (1.0 - aux["T_final"])[None], img_z[0:1], aux


def oracle_planes(means3D, opacities, cam, W, H, **kw):
    """The C oracle (float32) composed by the identities: (alpha (1,H,W), depth (1,H,W), the colour-free state).
    kw: scales / rotations / cov3D_precomp of orc.forward."""
    a = (means3D, opacities, cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
         cam.camera_center.numpy(), W, H, cam.tanfovx, cam.tanfovy)
    P = np.asarray(means3D).shape[0]
    st = orc.forward(*a, np.zeros(3, np.float32), colors_precomp=np.zeros((P, 3), np.float32), **kw)
    zc = np.zeros((P, 3), np.float32)
    zc[:, 0] = st.depths
    st_z = orc.forward(*a, np.zeros(3, np.float32), colors_precomp=zc, **kw)
    return (np.float32(1.0) - st.final_T)[None], st_z.out_color[0:1], st
