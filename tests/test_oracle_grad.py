"""CPU: the oracle's hand-restated backward (stage 4/5 of splat_oracle.c) against two independent anchors
(SURVEY.md 8c): float64 autograd of the dense model, and float64 central finite differences of its forward."""
import numpy as np
import pytest
import torch

from oracle import dense64
from oracle import rasterizer as orc
from tests import adversarial_scenes as A
from tests import helpers as h


def _dense(scene, t64, m2, radii, **over):
    cam = scene["cam"]
    kw = dict(shs=t64.get("shs"), sh_degree=scene["sh_degree"], scales=t64.get("scales"), rotations=t64.get("rotations"))
    kw.update(over)
    return dense64.render(t64["means3D"], m2, t64["opacities"], cam.world_view_transform.double(),
                          cam.full_proj_transform.double(), cam.camera_center.double(), scene["W"], scene["H"],
                          cam.tanfovx, cam.tanfovy, scene["bg"].double(), radii=radii, **kw)


def _leaf64(scene, names):
    return {k: scene[k].double().clone().requires_grad_(True) for k in names}


@pytest.mark.parametrize("deg,seed,mod", [(3, 3, 1.0), (1, 5, 1.0), (0, 8, 1.0), (2, 11, 0.7)])
def test_oracle_backward_equals_float64_autograd(deg, seed, mod):
    P, W, H = 160, 48, 40
    scene = h.random_scene(P, W, H, sh_degree=deg, seed=seed, scale_shift=1.2)
    scene["means3D"][:, :2] *= 0.6
    cam = scene["cam"]
    kw = dict(shs=scene["shs"].numpy(), sh_degree=deg, scales=scene["scales"].numpy(), rotations=scene["rotations"].numpy(),
              scale_modifier=mod)
    st = orc.forward(scene["means3D"].numpy(), scene["opacities"].numpy(), cam.world_view_transform.numpy(),
                     cam.full_proj_transform.numpy(), cam.camera_center.numpy(), W, H, cam.tanfovx, cam.tanfovy,
                     scene["bg"].numpy(), **kw)
    t64 = _leaf64(scene, ("means3D", "opacities", "scales", "rotations", "shs"))
    m2 = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    img, _ = _dense(scene, t64, m2, torch.from_numpy(st.radii).long(), scale_modifier=mod)
    ke = A.knife_edges(st)
    h.assert_image_explained(st.out_color, img.detach().numpy(), ke["pixels"], "oracle image vs float64", tol=5e-6, cap=5e-6)
    gout = torch.randn(3, H, W, generator=torch.Generator().manual_seed(1))
    img.backward(gout.double())
    g = orc.backward(st, gout.numpy(), scene["means3D"].numpy(), cam.world_view_transform.numpy(),
                     cam.full_proj_transform.numpy(), cam.camera_center.numpy(), cam.tanfovx, cam.tanfovy,
                     scene["bg"].numpy(), **kw)
    for name, ref in [("means3D", t64["means3D"].grad), ("means2D", m2.grad), ("opacities", t64["opacities"].grad),
                      ("scales", t64["scales"].grad), ("rotations", t64["rotations"].grad), ("shs", t64["shs"].grad)]:
        h.assert_grad_explained(g[name], ref.numpy(), A.affected(ke, name), f"oracle dL/d{name}", rtol=0.0, atol_frac=2e-5, knife_allowed=3)


def test_oracle_backward_precomputed_routes():
    P, W, H = 120, 40, 40
    scene = h.random_scene(P, W, H, sh_degree=0, seed=21, scale_shift=1.2)
    scene["means3D"][:, :2] *= 0.5
    cam = scene["cam"]
    colors = torch.rand(P, 3, generator=torch.Generator().manual_seed(2))
    R = dense64.quat_to_R(scene["rotations"].double())
    s = scene["scales"].double()
    S = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    cov = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], dim=1).float().contiguous()
    args = (cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(), cam.camera_center.numpy())
    st = orc.forward(scene["means3D"].numpy(), scene["opacities"].numpy(), *args, W, H, cam.tanfovx, cam.tanfovy,
                     scene["bg"].numpy(), colors_precomp=colors.numpy(), cov3D_precomp=cov.numpy())
    t64 = {"means3D": scene["means3D"].double().requires_grad_(True), "opacities": scene["opacities"].double().requires_grad_(True)}
    c64, v64 = colors.double().requires_grad_(True), cov.double().requires_grad_(True)
    m2 = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    img, _ = _dense(scene, t64, m2, torch.from_numpy(st.radii).long(), shs=None, scales=None, rotations=None,
                    colors_precomp=c64, cov3D_precomp=v64)
    gout = torch.randn(3, H, W, generator=torch.Generator().manual_seed(3))
    img.backward(gout.double())
    g = orc.backward(st, gout.numpy(), scene["means3D"].numpy(), *args, cam.tanfovx, cam.tanfovy, scene["bg"].numpy())
    ke = A.knife_edges(st)
    h.assert_grad_explained(g["colors_precomp"], c64.grad.numpy(), A.affected(ke, "colors_precomp"), "dL/dcolors", rtol=0.0, atol_frac=2e-5, knife_allowed=3)
    h.assert_grad_explained(g["cov3D_precomp"], v64.grad.numpy(), A.affected(ke, "cov3D_precomp"), "dL/dcov3D", rtol=0.0, atol_frac=5e-5, knife_allowed=3)
    h.assert_grad_explained(g["means3D"], t64["means3D"].grad.numpy(), A.affected(ke, "means3D"), "dL/dmeans3D", rtol=0.0, atol_frac=5e-5, knife_allowed=3)


def test_oracle_gradient_against_float64_finite_differences():
    """Directional derivatives of the float64 dense FORWARD (no autograd involved) vs <oracle gradient, direction>."""
    P, W, H, deg = 60, 32, 32, 2
    scene = h.random_scene(P, W, H, sh_degree=deg, seed=31, scale_shift=1.4)
    scene["means3D"][:, :2] *= 0.4
    cam = scene["cam"]
    kw = dict(shs=scene["shs"].numpy(), sh_degree=deg, scales=scene["scales"].numpy(), rotations=scene["rotations"].numpy())
    args = (cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(), cam.camera_center.numpy())
    st = orc.forward(scene["means3D"].numpy(), scene["opacities"].numpy(), *args, W, H, cam.tanfovx, cam.tanfovy,
                     scene["bg"].numpy(), **kw)
    gout = torch.randn(3, H, W, generator=torch.Generator().manual_seed(5))
    g = orc.backward(st, gout.numpy(), scene["means3D"].numpy(), *args, cam.tanfovx, cam.tanfovy, scene["bg"].numpy(), **kw)
    radii = torch.from_numpy(st.radii).long()
    names = ("means3D", "opacities", "scales", "rotations", "shs")
    base = {k: scene[k].double() for k in names}
    m2 = torch.zeros(P, 3, dtype=torch.float64)

    def loss(t64):
        with torch.no_grad():
            img, _ = _dense(scene, t64, m2, radii)
        return float((img * gout.double()).sum())

    gen = torch.Generator().manual_seed(9)
    for name in names:
        d = torch.randn(base[name].shape, generator=gen, dtype=torch.float64)
        eps = 1e-6 * float(base[name].abs().mean() + 1e-3)
        plus = dict(base); plus[name] = base[name] + eps * d
        minus = dict(base); minus[name] = base[name] - eps * d
        fd = (loss(plus) - loss(minus)) / (2 * eps)
        an = float((torch.from_numpy(g[name]).double().reshape(d.shape) * d).sum())
        # threshold decisions (alpha < 1/255, T < 1e-4) are discontinuities: a rare flip inside +-eps is tolerated
        assert abs(fd - an) <= 2e-3 * (abs(fd) + abs(an)) + 1e-6, f"{name}: finite difference {fd} vs analytic {an}"
