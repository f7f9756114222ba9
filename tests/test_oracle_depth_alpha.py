"""CPU: the float64 alpha and depth planes (tests/planes64.py, from oracle/dense64.py) against the float32 C oracle
composed by the identities, and against central differences along random directions -- for every raw group of the
ACTIVATED inputs on the adversarial builders that reach the walk's edges (the T < 1e-4 stop, the 1/255 skip, the near
plane, tile borders), and for BOUND_RAW through the binding and the face frame.  These are the references the GPU
planes are held to (tests/test_gpu_depth_alpha.py)."""
import numpy as np
import pytest
import torch

from oracle import binding as ob
from tests import adversarial_scenes as A
from tests import helpers as h
from tests import planes64 as P64

CASES = ["saturating_stack", "faint", "near_plane", "tile_borders", ("saturating_stack", 17, 15), ("faint", 15, 17),
         ("near_plane", 1, 37), ("tile_borders", 33, 31)]
GROUPS = ("means3D", "opacities", "scales", "rotations", "shs")
EPS = 1e-7


def _case(c):
    return (c, None, None) if isinstance(c, str) else c


def _id(c):
    return c if isinstance(c, str) else "-".join(map(str, c))


def _cam64(cam):
    d = torch.float64
    return cam.world_view_transform.to(d), cam.full_proj_transform.to(d), cam.camera_center.to(d)


def _planes(sc, st, t64, m2):
    cam = sc["cam"]
    V, Pm, c = _cam64(cam)
    _, alpha, depth, aux = P64.render(t64["means3D"], m2, t64["opacities"], V, Pm, c, sc["W"], sc["H"], cam.tanfovx,
                                      cam.tanfovy, sc["bg"].double(), shs=t64["shs"], sh_degree=sc["sh_degree"],
                                      scales=t64["scales"], rotations=t64["rotations"],
                                      radii=torch.from_numpy(st.radii).long(), rect_xy=torch.from_numpy(st.xy),
                                      depths=torch.from_numpy(st.depths))
    return alpha, depth, aux


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_dense64_planes_equal_the_oracle_composition(case):
    name, W, H = _case(case)
    sc = A.build(name, W, H)
    st = h.oracle_forward(sc)
    P = sc["means3D"].shape[0]
    t64 = {k: sc[k].double() for k in GROUPS}
    alpha, depth, aux = _planes(sc, st, t64, torch.zeros(P, 3, dtype=torch.float64))
    a_o, d_o, st_o = P64.oracle_planes(sc["means3D"].numpy(), sc["opacities"].numpy(), sc["cam"], sc["W"], sc["H"],
                                       scales=sc["scales"].numpy(), rotations=sc["rotations"].numpy())
    assert np.array_equal(st_o.n_contrib, st.n_contrib), "the colours changed the walk"
    assert np.abs(alpha.numpy() - a_o).max() < 5e-6
    scale = max(1.0, float(np.abs(d_o).max()))
    assert np.abs(depth.numpy() - d_o).max() < 5e-6 * scale
    # alpha comes from the colour image's own background weight: T_final does not depend on the colours
    assert np.array_equal(st_o.final_T, st.final_T)
    if name == "saturating_stack":
        assert (a_o > 1 - 1e-2).sum() >= 20, "no saturated pixel"
    assert (a_o > 0).any() and (d_o > 0).any()


def _check_directions(name, loss, base, leaves, gen, order, P):
    """For every group: the autograd derivative along a random direction against the central difference.  A step
    that flips a discrete decision of the walk (a pair crossing 1/255 or the T < 1e-4 stop: the builders put pairs
    within float32 ulps of both) has no derivative there; the splats whose pairs flip are taken out of the direction
    (rows of a per-splat group; a group that is not per splat must not flip at all)."""
    L, aux0 = loss(base)
    keep0 = aux0["keep"]
    # the gradient the reference defines is not the derivative for two documented quirks (oracle/dense64.py): min(0.99,
    # alpha) passes the gradient straight through, and the guard band drops the clamp's t.z dependence.  Splats in
    # either regime are left out of the directions; the GPU tests hold them to dense64's autograd instead.
    quirk = aux0["guard_clamped"].any(dim=1)
    quirk[order[aux0["alpha_clamped"].any(dim=0)]] = True
    live = ~quirk
    assert live.sum() >= 5, "too few splats outside the non-analytic regimes"
    for k in base:
        u = torch.randn(base[k].shape, generator=gen, dtype=torch.float64)
        if base[k].shape[0] == P:
            u[quirk] = 0.0
        for _ in range(4):
            flipped = torch.zeros(P, dtype=torch.bool)
            for sgn in (1.0, -1.0):
                t = dict(base)
                t[k] = base[k] + sgn * EPS * u
                cols = (loss(t)[1]["keep"] != keep0).any(dim=0)
                flipped[order[cols]] = True
            if not flipped.any():
                break
            assert base[k].shape[0] == P, f"{k}: a step that is not per splat flipped the walk"
            u[flipped] = 0.0
        else:
            raise AssertionError(f"{k}: the step keeps flipping the walk")
        if base[k].shape[0] == P:
            assert (u.reshape(P, -1) != 0).any(dim=1).sum() >= 0.8 * live.sum(), f"{k}: most splats flip the walk"
        g = leaves[k].grad
        ad = 0.0 if g is None else float((g * u).sum())

        def f(sgn, k=k):
            t = dict(base)
            t[k] = base[k] + sgn * EPS * u
            return float(loss(t)[0])
        cd = (f(1.0) - f(-1.0)) / (2 * EPS)
        tol = 1e-5 * max(abs(cd), abs(ad)) + 1e-8 * max(1.0, abs(float(L)))   # float64 rounding of the difference
        print(f"[cd] {name} {k:<15s} autograd {ad:+.10e} central {cd:+.10e}")
        assert abs(ad - cd) <= tol, f"{k}: autograd {ad} vs central difference {cd}"


def _order(st):
    """Column j of dense64's (pixel, instance) tensors is splat order[j]: the stable sort of the pinned depths."""
    return torch.argsort(torch.from_numpy(st.depths).to(torch.float32), stable=True)


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_dense64_planes_match_central_differences(case):
    name, W, H = _case(case)
    sc = A.build(name, W, H)
    st = h.oracle_forward(sc)
    P = sc["means3D"].shape[0]
    gen = torch.Generator().manual_seed(3)
    ga = torch.randn((1, sc["H"], sc["W"]), generator=gen, dtype=torch.float64)
    gd = torch.randn((1, sc["H"], sc["W"]), generator=gen, dtype=torch.float64)
    base = {k: sc[k].double() for k in GROUPS}
    base["means2D"] = torch.zeros(P, 3, dtype=torch.float64)

    def loss(t):
        alpha, depth, aux = _planes(sc, st, t, t["means2D"])
        return (alpha * ga).sum() + (depth * gd).sum(), aux

    leaves = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    loss(leaves)[0].backward()
    assert leaves["shs"].grad is None or not leaves["shs"].grad.any(), "the planes do not depend on the colours"
    _check_directions(name, loss, base, leaves, gen, _order(st), P)


def _bound_planes(sc, st, leaves, verts):
    """BOUND_RAW in float64: the reference getters (oracle/binding.py) on the face frame of `verts`, then the planes."""
    p = sc["params"]
    b = p["binding"].long()
    fr = ob.update_mesh_properties(verts, sc["faces"])
    act = dict(means3D=ob.get_xyz(leaves["_xyz"], b, fr["face_center"], fr["face_orien_mat"], fr["face_scaling"]),
               scales=ob.get_scaling(leaves["_scaling"], b, fr["face_scaling"]),
               rotations=ob.get_rotation(leaves["_rotation"], b, fr["face_orien_quat"]),
               opacities=ob.get_opacity(leaves["_opacity"]),
               shs=ob.get_features(leaves["_features_dc"], leaves["_features_rest"]))
    P = b.shape[0]
    return _planes(dict(sc, means3D=None), st, act, torch.zeros(P, 3, dtype=torch.float64))


def test_bound_raw_planes_match_central_differences_through_the_binding():
    sc = h.avatar_scene(P=300, W=48, H=40, seed=4)
    act32, _, _, _ = h.avatar_activated(sc)
    st = h.oracle_forward(dict(sc, **{k: v.detach() for k, v in act32.items()}))
    p = sc["params"]
    names = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
    base = {k: p[k].double() for k in names}
    base["verts"] = sc["verts"].double()
    gen = torch.Generator().manual_seed(5)
    ga = torch.randn((1, sc["H"], sc["W"]), generator=gen, dtype=torch.float64)
    gd = torch.randn((1, sc["H"], sc["W"]), generator=gen, dtype=torch.float64)

    def loss(t):
        alpha, depth, aux = _bound_planes(sc, st, t, t["verts"])
        return (alpha * ga).sum() + (depth * gd).sum(), aux

    leaves = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    L, aux0 = loss(leaves)
    assert float((aux0["T_final"] < 0.5).sum()) >= 20, "the avatar covers too few pixels"
    L.backward()
    _check_directions("bound", loss, base, leaves, gen, _order(st), p["_xyz"].shape[0])
