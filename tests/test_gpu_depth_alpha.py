"""-m gpu: the alpha and depth planes of the blend (gab200_forward_depth_alpha / gab200_backward_depth_alpha,
rasterize_bound(depth_alpha=True), render_display(depth_alpha=True), GraphedRender(depth_alpha=True)).

The planes are checked against the existing, already validated forward and backward through identities, because
the colour is linear in the colour inputs and does not change the walk:
  * alpha = 1 - img[0] of a plain forward with colors_precomp = 0 and bg = (1, 1, 1)   (fmaf(T, 1, 0) = T);
  * depth = img[0] of a plain forward with colors_precomp[:, 0] = z and bg = 0, z = ((V[2] x + V[6] y) + V[10] z) +
    V[14] of bind_activate's means, op by op (preprocess.cu is built with --fmad=false, so z is the kernel's value);
  * the gradients of (colour, alpha, depth) are those of three plain backwards: the colour pass, an alpha pass with
    colours 0, bg = (-1, 0, 0) and dL/dimg[0] = dL/dalpha, and a depth pass with colours (z, 0, 0), bg = 0 and
    dL/dimg[0] = dL/ddepth, whose colour gradient reaches the parameters through z (torch autograd).
Forward comparisons are bit for bit; gradient comparisons use the assert_grad_tight gates (atomics reorder sums)."""
from types import SimpleNamespace

import pytest
import torch

from tests import helpers as h
from tests.test_gpu_camera_fov import _Sync, _dev_tanfov, _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NAMES = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


@pytest.fixture(autouse=True)
def default_policies():
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    prev = R._EXACT_BINNING, N.tune(N.TUNE_TILE_SORT)
    yield
    R.set_exact_binning(prev[0])
    N.tune(N.TUNE_TILE_SORT, prev[1])
    R.set_sync_policy("late")


def _scene(W, H, P, seed=0):
    return h.avatar_scene(P=P, W=W, H=H, seed=seed)


def _z_of(means, V):
    """The preprocess's t.z, op by op in fp32 (V = the 16 floats of the view matrix as the kernels read them)."""
    return ((V[2] * means[:, 0] + V[6] * means[:, 1]) + V[10] * means[:, 2]) + V[14]


def _torch_means(leaves, binding, fc, fR, fs):
    """scene/flame_gaussian_model.py's get_xyz in torch (differentiable, fp32)."""
    b = binding.long()
    return torch.bmm(fR[b], leaves[0][..., None]).squeeze(-1) * fs.reshape(-1, 1)[b] + fc[b]


def _inputs(sc, grad=False):
    from gaussianavatars_b200.rasterizer import face_frame
    p = sc["params"]
    leaves = [p[k].to(DEV).clone().requires_grad_(grad) for k in NAMES]
    verts = sc["verts"].to(DEV).clone().requires_grad_(grad)
    fc, fR, fs = face_frame(verts, sc["faces"].to(DEV))
    return leaves, verts, p["binding"].to(DEV), (fc, fR, fs)


def _settings(sc, cam, bg=None):
    return h.cuda_settings(dict(cam=cam, W=sc["W"], H=sc["H"], bg=sc["bg"] if bg is None else bg, sh_degree=3), DEV,
                           debug=False)


def _raster(rs, leaves, binding, frame, sync, tanfov=None, **kw):
    from gaussianavatars_b200.rasterizer import rasterize_bound
    fc, fR, fs = frame
    m2 = kw.pop("means2D", None)

    def go(hints):
        return rasterize_bound(rs, *leaves, binding=binding, face_center=fc, face_orien_mat=fR, face_scaling=fs,
                               means2D=m2, grad_sink=SimpleNamespace(_gab200_hints=hints), tanfov=tanfov, **kw)
    return sync(go)


def _check_forward(sc, cam, mode, tanfov=None):
    """Colour, display bytes, radii and visibility equal the plain forward's; alpha and depth equal the identities."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import bind_activate
    W, H = sc["W"], sc["H"]
    key = (DEV, W, H, sc["params"]["_xyz"].shape[0])
    with torch.no_grad():
        leaves, _, binding, frame = _inputs(sc)
        rs = _settings(sc, cam)
        P = leaves[0].shape[0]
        rgb_a = torch.empty((H, W, 3), dtype=torch.uint8, device=DEV)
        rgb_b = torch.empty_like(rgb_a)
        img, radii = _raster(rs, leaves, binding, frame, _Sync(mode, key), tanfov, rgb8=rgb_a)
        vis = R.visible_of(radii).clone()
        img2, radii2, alpha, depth = _raster(rs, leaves, binding, frame, _Sync(mode, key), tanfov, rgb8=rgb_b,
                                             depth_alpha=True)
        vis2 = R.visible_of(radii2).clone()
        torch.cuda.synchronize()
        assert alpha.shape == (1, H, W) and depth.shape == (1, H, W)
        assert torch.equal(img, img2) and torch.equal(rgb_a, rgb_b), "the colour image changed"
        assert torch.equal(radii, radii2) and torch.equal(vis, vis2), "radii / visibility changed"
        # alpha: colours 0 over a white background leave T_final in every channel
        zero = torch.zeros((P, 3), device=DEV)
        white = _settings(sc, cam, torch.ones(3))
        img_t, _ = _raster(white, leaves, binding, frame, _Sync(mode, key), tanfov, colors_precomp=zero)
        assert torch.equal(alpha, 1.0 - img_t[0:1]), "alpha != 1 - T_final"
        # depth: the colour channel 0 carrying z over a black background
        means = bind_activate(rs, *leaves[:4], binding, *frame)[0]
        z = _z_of(means, rs.viewmatrix.reshape(-1))
        zc = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], 1).contiguous()
        black = _settings(sc, cam, torch.zeros(3))
        img_z, _ = _raster(black, leaves, binding, frame, _Sync(mode, key), tanfov, colors_precomp=zc)
        assert torch.equal(depth, img_z[0:1]), "depth != sum w z"
        return alpha, depth


@pytest.mark.parametrize("mode", ["exact", "late", "none"])
@pytest.mark.parametrize("exact_binning", [False, True])
@pytest.mark.parametrize("tile_sort", [0, 1])
def test_forward_planes_match_the_identities(mode, exact_binning, tile_sort):
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    R.set_exact_binning(exact_binning)
    N.tune(N.TUNE_TILE_SORT, tile_sort)
    sc = _scene(192, 160, 6000, seed=1)
    cam = _rig(sc["W"], sc["H"], n=4)[1]
    alpha, depth = _check_forward(sc, cam, mode, _dev_tanfov(cam))
    assert float(alpha.max()) > 0.5 and float(depth.max()) > 0.0, "the scene draws nothing"


@pytest.mark.parametrize("W,H", [(1, 1), (1, 37), (37, 1), (15, 17), (17, 15), (33, 31), (4, 20)])
def test_forward_planes_at_ragged_sizes(W, H):
    sc = _scene(W, H, 3000, seed=2)
    cam = _rig(W, H, n=4)[2]
    _check_forward(sc, cam, "exact")
    _check_forward(sc, cam, "none")


def test_forward_planes_at_1080p_with_long_tile_lists():
    import gaussianavatars_b200.rasterizer as R
    sc = _scene(1920, 1080, 100_000, seed=3)
    cam = _rig(1920, 1080, n=4)[1]
    R.keep_last_state(True)
    try:
        _check_forward(sc, cam, "exact")
        _, _, ranges, _ = R.export_last_binning()
    finally:
        R.keep_last_state(False)
    longest = int((ranges[:, 1] - ranges[:, 0]).max())
    print(f"[1080p] longest tile list {longest}")
    assert longest > 2048


def test_invalid_fov_gives_empty_planes():
    sc = _scene(64, 48, 2000, seed=4)
    cam = _rig(64, 48, n=4)[0]
    bad = torch.tensor([0.0, float("nan")], device=DEV)
    alpha, depth = _check_forward(sc, cam, "exact", bad)
    assert not alpha.any() and not depth.any()


@pytest.mark.parametrize("name", ["needles", "near_plane", "guard_band", "saturating_stack", "faint",
                                  "tile_borders+ties", "guard_band+sh3"])
def test_forward_planes_on_adversarial_scenes(name):
    """The adversarial builders as a plain GaussianModel (binding=None, the identity frame): raw parameters whose
    getters give the builder's activated values."""
    from gaussianavatars_b200.rasterizer import rasterize_bound
    from tests import adversarial_scenes as A
    sc = A.build(name)
    W, H = sc["W"], sc["H"]
    P = sc["means3D"].shape[0]
    shs = sc["shs"].to(DEV)
    leaves = [sc["means3D"].to(DEV), sc["rotations"].to(DEV), torch.log(sc["scales"].to(DEV)),
              torch.logit(sc["opacities"].to(DEV).double()).float(), shs[:, :1].contiguous(),
              shs[:, 1:].contiguous() if shs.shape[1] > 1 else None]
    rs = h.cuda_settings(dict(cam=sc["cam"], W=W, H=H, bg=sc["bg"], sh_degree=sc["sh_degree"]), DEV, debug=False)
    with torch.no_grad():
        img, radii = rasterize_bound(rs, *leaves)
        img2, radii2, alpha, depth = rasterize_bound(rs, *leaves, depth_alpha=True)
        assert torch.equal(img, img2) and torch.equal(radii, radii2)
        white = h.cuda_settings(dict(cam=sc["cam"], W=W, H=H, bg=torch.ones(3), sh_degree=sc["sh_degree"]), DEV,
                                debug=False)
        img_t, _ = rasterize_bound(white, *leaves, colors_precomp=torch.zeros((P, 3), device=DEV))
        assert torch.equal(alpha, 1.0 - img_t[0:1])
        from gaussianavatars_b200.rasterizer import bind_activate
        means = bind_activate(rs, *leaves[:4])[0]
        z = _z_of(means, rs.viewmatrix.reshape(-1))
        black = h.cuda_settings(dict(cam=sc["cam"], W=W, H=H, bg=torch.zeros(3), sh_degree=sc["sh_degree"]), DEV,
                                debug=False)
        zc = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], 1).contiguous()
        img_z, _ = rasterize_bound(black, *leaves, colors_precomp=zc)
        assert torch.equal(depth, img_z[0:1])


# ---- backward ---------------------------------------------------------------------------------------------------
def _grads(sc, cam, loss_fn, depth_alpha=False, bg=None, colors=None, seed=0, mode="exact"):
    """One differentiable frame; loss_fn(out) -> scalar.  colors: None, "zero" or "z" (z from the torch binding)."""
    leaves, verts, binding, frame = _inputs(sc, grad=True)
    rs = _settings(sc, cam, bg)
    P = leaves[0].shape[0]
    m2 = torch.zeros((P, 3), device=DEV, requires_grad=True)
    cp = None
    if colors == "zero":
        cp = torch.zeros((P, 3), device=DEV)
    elif colors == "z":
        z = _z_of(_torch_means(leaves, binding, *frame), rs.viewmatrix.reshape(-1))
        cp = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], 1)
    key = (DEV, sc["W"], sc["H"], P)
    out = _raster(rs, leaves, binding, frame, _Sync(mode, key), _dev_tanfov(cam), means2D=m2, colors_precomp=cp,
                  depth_alpha=depth_alpha)
    loss_fn(out).backward()
    torch.cuda.synchronize()
    g = [x.grad if x.grad is not None else torch.zeros_like(x) for x in leaves if x is not None]
    return g + [m2.grad, verts.grad], out[1]


def _check_backward(sc, cam, seed=5, mode="exact"):
    W, H = sc["W"], sc["H"]
    gen = torch.Generator().manual_seed(seed)
    gc = torch.randn((3, H, W), generator=gen).to(DEV)
    ga = torch.randn((1, H, W), generator=gen).to(DEV)
    gd = torch.randn((1, H, W), generator=gen).to(DEV) * 0.5
    full, radii = _grads(sc, cam, lambda o: (o[0] * gc).sum() + (o[2] * ga).sum() + (o[3] * gd).sum(), True,
                         mode=mode)
    col, _ = _grads(sc, cam, lambda o: (o[0] * gc).sum())
    alp, _ = _grads(sc, cam, lambda o: (o[0][0:1] * ga).sum(), bg=torch.tensor([-1.0, 0.0, 0.0]), colors="zero")
    dep, _ = _grads(sc, cam, lambda o: (o[0][0:1] * gd).sum(), bg=torch.zeros(3), colors="z")
    names = list(NAMES[:len(full) - 2]) + ["means2D", "verts"]
    for n, g, a, b, c in zip(names, full, col, alp, dep):
        ref = (a.double() + b.double() + c.double()).cpu().numpy()
        h.assert_grad_tight(g.double().cpu().numpy(), ref, f"{n} (colour+alpha+depth)")
    # only the depth and alpha terms: the three-term sum must not be carried by the colour pass alone
    assert (full[0] - col[0]).abs().max() > 0
    # splats without an instance get exactly zero gradient
    dead = radii == 0
    if bool(dead.any()):
        for n, g in zip(names[:4], full[:4]):
            assert not g[dead].any(), f"{n}: a culled splat received a gradient"
    return full


@pytest.mark.parametrize("mode", ["exact", "late", "none"])
def test_backward_is_the_sum_of_three_plain_backwards(mode):
    """Under every sync mode of the depth-alpha forward (NONE: the state's num_rendered is -1)."""
    sc = _scene(192, 160, 6000, seed=6)
    cam = _rig(sc["W"], sc["H"], n=4)[2]
    full = _check_backward(sc, cam, mode=mode)
    assert float(full[-1].abs().max()) > 0, "no gradient reached the vertices"


@pytest.mark.parametrize("W,H", [(15, 17), (33, 31), (4, 20)])
def test_backward_at_ragged_sizes(W, H):
    sc = _scene(W, H, 2000, seed=7)
    _check_backward(sc, _rig(W, H, n=4)[1])


def test_backward_at_1080p():
    sc = _scene(1920, 1080, 100_000, seed=8)
    _check_backward(sc, _rig(1920, 1080, n=4)[1])


def test_plain_backward_on_a_depth_alpha_state_is_the_colour_backward(monkeypatch):
    """gab200_backward (not gab200_backward_depth_alpha) on the state a depth-alpha forward kept: the colour backward."""
    import gaussianavatars_b200.rasterizer as R
    sc = _scene(96, 80, 3000, seed=9)
    cam = _rig(96, 80, n=4)[0]
    W, H = sc["W"], sc["H"]
    gc = torch.randn((3, H, W), generator=torch.Generator().manual_seed(1)).to(DEV)
    calls = []
    run = R._run_backward

    def plain_backward(b, device, tanfov=None, plane_grads=None):
        calls.append(plane_grads)
        assert b.state.contents.depth_prefix == 1, "not a depth-alpha state"
        return run(b, device, tanfov, None)   # gab200_backward_device_fov, the plain entry point
    monkeypatch.setattr(R, "_run_backward", plain_backward)
    da, _ = _grads(sc, cam, lambda o: (o[0] * gc).sum(), True)
    monkeypatch.setattr(R, "_run_backward", run)
    assert len(calls) == 1 and calls[0] is not None
    plain, _ = _grads(sc, cam, lambda o: (o[0] * gc).sum())
    for g, r in zip(da, plain):
        h.assert_grad_tight(g.double().cpu().numpy(), r.double().cpu().numpy(), "colour only")


# ---- against the C oracle and float64 ----------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(15, 17), (17, 15), (33, 31), (4, 20), (1, 37)])
@pytest.mark.parametrize("name", ["saturating_stack", "faint", "near_plane", "tile_borders"])
def test_planes_and_gradients_against_the_oracle_and_float64_at_ragged_sizes(name, W, H):
    """Plain GaussianModel inputs (binding=None): the planes against the C-oracle composition (tests/planes64.py),
    dL/d_xyz and dL/dmeans2D of <alpha, ga> + <depth, gd> against float64 autograd of the dense model."""
    from tests import adversarial_scenes as A
    planes_against_the_oracle_and_float64(A.build(name, W, H), f"{name} {W}x{H}")


def planes_against_the_oracle_and_float64(sc, what):
    """The check of the test above on the activated scene `sc`, under the explained gates of tests/helpers.py (the
    knife set of adversarial_scenes.knife_edges on the oracle's state)."""
    from gaussianavatars_b200.rasterizer import bind_activate, rasterize_bound
    from tests import adversarial_scenes as A
    from tests import planes64 as P64
    W, H = sc["W"], sc["H"]
    P = sc["means3D"].shape[0]
    shs = sc["shs"].to(DEV)
    leaves = [sc["means3D"].to(DEV).clone().requires_grad_(True), sc["rotations"].to(DEV),
              torch.log(sc["scales"].to(DEV)), torch.logit(sc["opacities"].to(DEV).double()).float(),
              shs[:, :1].contiguous(), shs[:, 1:].contiguous() if shs.shape[1] > 1 else None]
    rs = h.cuda_settings(dict(cam=sc["cam"], W=W, H=H, bg=sc["bg"], sh_degree=sc["sh_degree"]), DEV, debug=False)
    m2 = torch.zeros((P, 3), device=DEV, requires_grad=True)
    _, _, alpha, depth = rasterize_bound(rs, *leaves, means2D=m2, depth_alpha=True)
    gen = torch.Generator().manual_seed(2)
    ga, gd = torch.randn((1, H, W), generator=gen), torch.randn((1, H, W), generator=gen)
    ((alpha * ga.to(DEV)).sum() + (depth * gd.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    with torch.no_grad():
        m, op, s, _ = bind_activate(rs, *[x.detach() if x is not None else None for x in leaves[:4]])
    rot = sc["rotations"] / sc["rotations"].norm(dim=1, keepdim=True)   # the BOUND_RAW getter normalises
    act = dict(means3D=m.cpu(), opacities=op.cpu(), scales=s.cpu(), rotations=rot.contiguous())
    a_o, d_o, st = P64.oracle_planes(act["means3D"].numpy(), act["opacities"].numpy(), sc["cam"], W, H,
                                     scales=act["scales"].numpy(), rotations=act["rotations"].numpy())
    ke = A.knife_edges(st)
    print(f"[knife] {what}: {ke['pairs']} pairs, {int(ke['pixels'].sum())} pixels, {int(ke['splats'].sum())}/{P} "
          f"splats, {int(ke['ill'].sum())} ill-conditioned")
    h.assert_image_explained(alpha.detach().cpu().numpy(), a_o, ke["pixels"], f"{what}: alpha vs oracle")
    dscale = max(1.0, float(abs(d_o).max()))
    h.assert_image_explained(depth.detach().cpu().numpy() / dscale, d_o / dscale, ke["pixels"],
                             f"{what}: depth vs oracle")
    cam = sc["cam"]
    t64 = {k: v.double().clone().requires_grad_(k == "means3D") for k, v in act.items()}
    m64 = torch.zeros((P, 3), dtype=torch.float64, requires_grad=True)
    _, a64, d64, _ = P64.render(t64["means3D"], m64, t64["opacities"], cam.world_view_transform.double(),
                                cam.full_proj_transform.double(), cam.camera_center.double(), W, H, cam.tanfovx,
                                cam.tanfovy, sc["bg"].double(), shs=sc["shs"].double(), sh_degree=sc["sh_degree"],
                                scales=t64["scales"], rotations=t64["rotations"],
                                radii=torch.from_numpy(st.radii).long(), rect_xy=torch.from_numpy(st.xy),
                                depths=torch.from_numpy(st.depths))
    ((a64 * ga.double()).sum() + (d64 * gd.double()).sum()).backward()
    h.assert_grad_explained(leaves[0].grad.double().cpu().numpy(), t64["means3D"].grad.numpy(),
                            A.affected(ke, "_xyz"), f"{what}: _xyz")
    h.assert_grad_explained(m2.grad.double().cpu().numpy(), m64.grad.numpy(), A.affected(ke, "means2D"),
                            f"{what}: means2D")


def test_depth_and_alpha_gradients_reach_the_flame_parameters():
    """A BOUND_RAW head posed by FLAME on the device, <alpha, ga> + <depth, gd> through eager autograd into the posed
    FLAME rows, against central differences of the float64 composition of tests/train_step_oracle.py's pieces
    (FLAME -> face frame -> getters -> the dense planes, decisions pinned to the float32 C oracle)."""
    from oracle import binding as ob
    from oracle.fused_reference import RAW
    from gaussianavatars_b200.renderer import render
    from tests import flame_oracle as fo
    from tests import planes64 as P64
    from tests import train_step_oracle as T
    from tests.test_gpu_train_step import _model
    sc = T.scene(P=1500, W=64, H=48)
    t, W, H, cam = 2, sc["W"], sc["H"], sc["cam"]
    fl = T.flags(3)
    pc = _model(sc, 3)
    pc.select_mesh_by_timestep(t)
    out = render(cam.to(DEV), pc, Pipe, torch.tensor(fl["bg"], device=DEV), depth_alpha=True)
    gen = torch.Generator().manual_seed(4)
    ga, gd = torch.randn((1, H, W), generator=gen), torch.randn((1, H, W), generator=gen)
    ((out["alpha"] * ga.to(DEV)).sum() + (out["depth"] * gd.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    lib = {k: pc.flame_param[k].grad[t].double().cpu() for k in fo.POSED}

    faces = sc["assets"]["faces"].long()
    b = sc["params"]["binding"].long()

    def activation(fp, dtype):
        a = fo.assets_as({k: sc["assets"][k] for k in ("v_template", "shapedirs", "posedirs", "J_regressor",
                                                       "lbs_weights", "parents")}, dtype)
        verts = fo.select_mesh_by_timestep(a, fp, t)[0][0]
        fr = ob.update_mesh_properties(verts, faces)
        leaves = {k: sc["params"][k].to(dtype) for k in RAW}
        return dict(means3D=ob.get_xyz(leaves["_xyz"], b, fr["face_center"], fr["face_orien_mat"], fr["face_scaling"]),
                    scales=ob.get_scaling(leaves["_scaling"], b, fr["face_scaling"]),
                    rotations=ob.get_rotation(leaves["_rotation"], b, fr["face_orien_quat"]),
                    opacities=ob.get_opacity(leaves["_opacity"]),
                    shs=ob.get_features(leaves["_features_dc"], leaves["_features_rest"]))

    fp32 = {k: v.float() for k, v in sc["flame_param"].items() if v is not None and k != "dynamic_offset"}
    a32 = activation(fp32, torch.float32)
    st = T.oracle_forward_on(a32["means3D"], a32["opacities"], cam, W, H, fl, a32["shs"], a32["scales"],
                             a32["rotations"])
    vis = torch.from_numpy(st.radii) > 0
    d = torch.float64

    def loss64(fp):
        act = activation(fp, d)
        P = act["means3D"].shape[0]
        _, a64, d64, _ = P64.render(act["means3D"][vis], torch.zeros((P, 3), dtype=d)[vis], act["opacities"][vis],
                                    cam.world_view_transform.to(d), cam.full_proj_transform.to(d),
                                    cam.camera_center.to(d), W, H, cam.tanfovx, cam.tanfovy,
                                    torch.tensor(fl["bg"], dtype=d), shs=act["shs"][vis], sh_degree=3,
                                    scales=act["scales"][vis], rotations=act["rotations"][vis],
                                    radii=torch.from_numpy(st.radii).long()[vis], rect_xy=torch.from_numpy(st.xy)[vis],
                                    depths=torch.from_numpy(st.depths)[vis])
        return (a64 * ga.double()).sum() + (d64 * gd.double()).sum()

    base = {k: v.double() for k, v in fp32.items()}
    eps = 1e-6
    for k in fo.POSED:
        u = torch.zeros_like(base[k])
        u[t] = torch.randn(base[k].shape[1], generator=gen, dtype=d)
        plus, minus = dict(base), dict(base)
        plus[k], minus[k] = base[k] + eps * u, base[k] - eps * u
        cd = float((loss64(plus) - loss64(minus)) / (2 * eps))
        got = float((lib[k] * u[t]).sum())
        print(f"[flame] {k:<12s} library {got:+.6e} central difference {cd:+.6e}")
        assert abs(got - cd) <= 5e-3 * abs(cd) + 1e-4 * float(lib[k].norm() * u[t].norm()), k
    assert any(float(lib[k].abs().max()) > 0 for k in fo.POSED)



# ---- playback -----------------------------------------------------------------------------------------------------
def test_graphed_render_refreshes_the_planes_without_recapture():
    from gaussianavatars_b200.graph import GraphedRender
    from gaussianavatars_b200.renderer import render_display
    from tests.test_gpu_display import _flame_setup
    W, H = 400, 304
    pc = _flame_setup(T=6)
    cams = _rig(W, H, n=4)
    bg = torch.ones(3)
    view = GraphedRender(pc, W, H, bg, outputs="both", warm_cameras=cams, warm_timesteps=range(6), depth_alpha=True)

    def same(cam, t, bgv, what):
        torch.cuda.synchronize()
        pc.select_mesh_by_timestep(t)
        ref = render_display(cam, pc, Pipe, bgv.to(DEV), float_image=True, depth_alpha=True)
        torch.cuda.synchronize()
        for k, v in (("render", view.image), ("display_u8", view.display), ("radii", view.radii),
                     ("alpha", view.alpha), ("depth", view.depth)):
            assert torch.equal(v, ref[k]), f"{what}: {k} differs"

    for i, cam in enumerate(cams):
        view.set_inputs(camera=cam, timestep=(2 * i) % 6)
        view.run(check=True)
        same(cam, (2 * i) % 6, bg, f"camera {i}")
    bg2 = torch.tensor([0.2, 0.5, 0.9])
    view.set_inputs(camera=cams[1], timestep=3, bg=bg2.to(DEV))
    view.run(check=True)
    same(cams[1], 3, bg2, "background")
    assert view.captures == 1 and not view.overflowed()
    # an overflowed replay is flagged as without the planes
    small = GraphedRender(pc, W, H, bg, outputs="u8", capacity=2000, depth_alpha=True)
    small.set_inputs(camera=cams[2], timestep=1)
    small.run(check=False)
    assert small.overflowed()
    small.run(check=True)
    assert not small.overflowed()
    torch.cuda.synchronize()
    pc.select_mesh_by_timestep(1)
    ref = render_display(cams[2], pc, Pipe, bg.to(DEV), depth_alpha=True)
    assert torch.equal(small.alpha, ref["alpha"]) and torch.equal(small.depth, ref["depth"])
    assert torch.equal(small.display, ref["display_u8"])
