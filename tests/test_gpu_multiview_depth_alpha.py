"""-m gpu: the alpha and depth planes of a K-view frame (gab200_forward_views_depth_alpha,
gab200_forward_views_train_depth_alpha, gab200_backward_views_depth_alpha; rasterize_bound_views[_train](...,
depth_alpha=True), render_views[_train](..., depth_alpha=True)) on the mesh-bound rigs of tests/bound_rigs.py, where
one splat sits at a different edge in each view and view 5 has an invalid field of view.

    forward     colour, display bytes, radii, visibility, alpha and depth of both K-view forms equal K single-view
                gab200_forward_depth_alpha frames (each with its own tanfov) bit for bit, and colour and radii equal
                the plane-less K-view forwards -- under EXACT / LATE (re-enqueued) / NONE, both binnings, both tile
                sorts, the ragged sizes and 1080p with tile lists beyond 2048
    backward    for <image, gc> + <alpha, ga> + <depth, gd> summed over the views: the six raw groups, the face frame,
                dL/dverts and every (k, P, 3) dL/dmeans2D row against the sum of K single-view
                gab200_backward_depth_alpha steps, under assert_grad_tight with no outliers; culled splats get zeros
    plain       gab200_backward_views on a K-view depth-alpha state is the plain K-view colour backward
    float64     planes against the C oracle composed by tests/planes64.py, and the summed gradients against
                tests/planes64.py's float64 planes per view, pinned to that view's oracle decisions, at ragged sizes
    FLAME       the plane gradients of a K-view frame reach the posed FLAME rows as the sum of single-view frames do
The gradient comparisons use gates, not bit equality: the blend backward adds its per-splat gradients with atomics."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import bound_rigs as B
from tests import helpers as h
from tests import train_step_oracle as T
from tests.test_gpu_multiview_adversarial import _case, _gate_all, _leaves, _settings

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
STRICT = dict(max_outlier_frac=0.0, min_outliers_allowed=0)


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


@pytest.fixture(autouse=True)
def default_policies():
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    prev = R._EXACT_BINNING, R._SYNC_POLICY, N.tune(N.TUNE_TILE_SORT)
    yield
    R.set_exact_binning(prev[0])
    R.set_sync_policy(prev[1])
    N.tune(N.TUNE_TILE_SORT, prev[2])


def _run(mode, key, fn):
    """fn(hints) under one sync mode; LATE with a one-instance capacity, so the frame is always re-enqueued and the
    re-enqueued blend is the one whose planes are compared."""
    import gaussianavatars_b200.rasterizer as R
    hints = R.FrameHints()
    R.set_sync_policy("exact" if mode == "exact" else "late")
    try:
        if mode == "late":
            hints.set_capacity(key, 1)
            hints.set_depth(key, (0, 0))
        if mode == "none":
            R._capture_slot = R.CaptureSlot(DEV, 4_000_000)
        out = fn(hints)
    finally:
        R._capture_slot = None
        R.set_sync_policy("late")
    if mode == "late" and hints.last["num_rendered"] > 1:
        assert hints.last["attempts"] == 2 and hints.last["sync_mode"] == 1
    return out


def _rig(bound, K):
    cams = B.rig(bound, K)
    return cams, B.table(cams, DEV)


def _planes_of_singles(bound, table, mode, leaves, frame):
    """K single-view depth-alpha frames, each with its camera row's own field of view."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import rasterize_bound
    W, H = bound["W"], bound["H"]
    P = leaves["_xyz"].shape[0]
    binding = bound["params"]["binding"].to(DEV)
    out = []
    for k in range(table.shape[0]):
        row = table[k]
        rgb8 = torch.empty((H, W, 3), dtype=torch.uint8, device=DEV)
        img, radii, alpha, depth = _run(mode, (DEV, W, H, P), lambda hints: rasterize_bound(
            _settings(bound, row), *(leaves[n] for n in B.RAW), binding, *frame,
            grad_sink=SimpleNamespace(_gab200_hints=hints), tanfov=row[35:37].clone(), rgb8=rgb8, depth_alpha=True))
        out.append(dict(img=img, rgb8=rgb8, radii=radii, vis=R.visible_of(radii).clone(), alpha=alpha, depth=depth))
    return out


def _check_forward(bound, K, mode, what):
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound_views, rasterize_bound_views_train
    W, H = bound["W"], bound["H"]
    _, table = _rig(bound, K)
    with torch.no_grad():
        leaves = {n: t.detach() for n, t in _leaves(bound)[0].items()}
        frame = face_frame(bound["verts"].to(DEV), bound["faces"].to(DEV))
        binding = bound["params"]["binding"].to(DEV)
        P = leaves["_xyz"].shape[0]
        args = (_settings(bound), table, *(leaves[n] for n in B.RAW), binding, *frame)
        key = (DEV, W, H, P, K)
        singles = _planes_of_singles(bound, table, mode, leaves, frame)
        img, rgb8, radii, vis, alpha, depth = _run(mode, key, lambda hints: rasterize_bound_views(
            *args, hints=hints, display=True, float_image=True, depth_alpha=True))
        img_t, radii_t, alpha_t, depth_t = _run(mode, key, lambda hints: rasterize_bound_views_train(
            *args, hints=hints, depth_alpha=True))
        vis_t = R.visible_of(radii_t).clone()
        img_p, rgb8_p, radii_p, vis_p = rasterize_bound_views(*args, hints=R.FrameHints(), display=True,
                                                              float_image=True)
        img_pt, radii_pt = rasterize_bound_views_train(*args, hints=R.FrameHints())
        torch.cuda.synchronize()
    assert alpha.shape == depth.shape == alpha_t.shape == depth_t.shape == (K, 1, H, W)
    for k, s in enumerate(singles):
        for name, got in (("image", img), ("train image", img_t)):
            assert torch.equal(got[k], s["img"]), f"{what}: view {k} {name} differs from its single view"
        assert torch.equal(rgb8[k], s["rgb8"]), f"{what}: view {k} display bytes differ"
        for name, got in (("radii", radii), ("train radii", radii_t)):
            assert torch.equal(got[k], s["radii"]), f"{what}: view {k} {name} differ"
        for name, got in (("visibility", vis), ("train visibility", vis_t)):
            assert torch.equal(got[k], s["vis"]), f"{what}: view {k} {name} differs"
        for name, got in (("alpha", alpha), ("train alpha", alpha_t)):
            assert torch.equal(got[k], s["alpha"]), f"{what}: view {k} {name} differs from its single view"
        for name, got in (("depth", depth), ("train depth", depth_t)):
            assert torch.equal(got[k], s["depth"]), f"{what}: view {k} {name} differs from its single view"
        if not B.valid(k):
            assert not alpha[k].any() and not depth[k].any(), f"{what}: the invalid-FoV view has planes"
    assert torch.equal(img, img_p) and torch.equal(rgb8, rgb8_p) and torch.equal(radii, radii_p)
    assert torch.equal(vis, vis_p), f"{what}: visibility changed with the planes"
    assert torch.equal(img_t, img_pt) and torch.equal(radii_t, radii_pt), f"{what}: the train form changed"
    return alpha, depth


# ---- 1. forward, bit for bit ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["exact", "late", "none"])
@pytest.mark.parametrize("exact_binning", [False, True])
@pytest.mark.parametrize("tile_sort", [0, 1])
@pytest.mark.parametrize("name", ["near_plane", "saturating_stack"])
def test_forward_planes_every_sync_mode_and_schedule(name, mode, exact_binning, tile_sort):
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    R.set_exact_binning(exact_binning)
    N.tune(N.TUNE_TILE_SORT, tile_sort)
    bound = _case((name, None, None))["bound"]
    alpha, _ = _check_forward(bound, 3, mode, f"{name} K=3 {mode} exact={exact_binning} tile_sort={tile_sort}")
    assert float(alpha.max()) > 0.5, "the rig draws nothing"


@pytest.mark.parametrize("K", [1, 2, 6])
@pytest.mark.parametrize("name", ["needles", "near_plane", "guard_band+sh3", "faint"])
def test_forward_planes_other_view_counts(name, K):
    _check_forward(_case((name, None, None))["bound"], K, "exact", f"{name} K={K}")


@pytest.mark.parametrize("W,H", [(1, 37), (15, 17), (33, 31), (4, 20)])
@pytest.mark.parametrize("name", ["saturating_stack", "tile_borders"])
def test_forward_planes_at_ragged_sizes(name, W, H):
    bound = _case((name, W, H))["bound"]
    _check_forward(bound, 6, "exact", f"{name} {W}x{H}")
    _check_forward(bound, 6, "none", f"{name} {W}x{H} none")


def test_forward_planes_at_1080p_with_long_tile_lists():
    """An avatar scene at 1920x1080, two cameras: the tile lists run beyond 2048 entries."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound, rasterize_bound_views
    from gaussianavatars_b200.renderer import camera_table
    from tests.test_gpu_camera_fov import _rig as orbit_rig
    sc = h.avatar_scene(P=100_000, W=1920, H=1080, seed=3)
    W, H = sc["W"], sc["H"]
    table = camera_table(orbit_rig(W, H, n=4)[1:3], DEV)
    p = sc["params"]
    with torch.no_grad():
        leaves = [p[k].to(DEV) for k in B.RAW]
        frame = face_frame(sc["verts"].to(DEV), sc["faces"].to(DEV))
        binding = p["binding"].to(DEV)
        bound = dict(bg=sc["bg"], H=H, W=W, sh_degree=3)
        R.keep_last_state(True)
        try:
            singles = []
            for k in range(2):
                singles.append(rasterize_bound(_settings(bound, table[k]), *leaves, binding, *frame,
                                               tanfov=table[k, 35:37].clone(), depth_alpha=True))
                _, _, ranges, _ = R.export_last_binning()
                longest = int((ranges[:, 1] - ranges[:, 0]).max())
                print(f"[1080p] view {k}: longest tile list {longest}")
                assert longest > 2048
        finally:
            R.keep_last_state(False)
        img, _, radii, _, alpha, depth = rasterize_bound_views(_settings(bound), table, *leaves, binding, *frame,
                                                               display=False, float_image=True, depth_alpha=True)
        torch.cuda.synchronize()
    for k, (s_img, s_radii, s_alpha, s_depth) in enumerate(singles):
        assert torch.equal(img[k], s_img) and torch.equal(radii[k], s_radii)
        assert torch.equal(alpha[k], s_alpha) and torch.equal(depth[k], s_depth), f"1080p view {k}: planes differ"


# ---- 2. backward against K single-view backwards ---------------------------------------------------------------------
def _upstream(bound, K, seed=7):
    g = torch.Generator().manual_seed(seed)
    W, H = bound["W"], bound["H"]
    return (torch.randn((K, 3, H, W), generator=g).to(DEV), torch.randn((K, 1, H, W), generator=g).to(DEV),
            (0.5 * torch.randn((K, 1, H, W), generator=g)).to(DEV))


def _step(bound, table, gc, ga, gd, views, mode="exact"):
    """One step on fresh leaves: the K-view frame (views=True) or K single-view frames (False), loss
    <image, gc> + <alpha, ga> + <depth, gd> over the views.  Returns the gradients as float64 numpy."""
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound, rasterize_bound_views_train
    K = table.shape[0]
    W, H = bound["W"], bound["H"]
    leaves, verts = _leaves(bound)
    fc, fR, fs = face_frame(verts, bound["faces"].to(DEV))
    for t in (fc, fR, fs):
        t.retain_grad()
    binding = bound["params"]["binding"].to(DEV)
    P = leaves["_xyz"].shape[0]
    raw = [leaves[n] for n in B.RAW]
    if views:
        m2d = torch.zeros((K, P, 3), device=DEV, requires_grad=True)
        img, radii, alpha, depth = _run(mode, (DEV, W, H, P, K), lambda hints: rasterize_bound_views_train(
            _settings(bound), table, *raw, binding, fc, fR, fs, means2D=m2d, hints=hints, depth_alpha=True))
        ((img * gc).sum() + (alpha * ga).sum() + (depth * gd).sum()).backward()
        rows = m2d.grad
    else:
        rows, radii = [], []
        for k in range(K):
            m2 = torch.zeros((P, 3), device=DEV, requires_grad=True)
            img, r, alpha, depth = _run(mode, (DEV, W, H, P), lambda hints: rasterize_bound(
                _settings(bound, table[k]), *raw, binding, fc, fR, fs, means2D=m2,
                grad_sink=SimpleNamespace(_gab200_hints=hints), tanfov=table[k, 35:37].clone(), depth_alpha=True))
            ((img * gc[k]).sum() + (alpha * ga[k]).sum() + (depth * gd[k]).sum()).backward(retain_graph=True)
            rows.append(m2.grad)
            radii.append(r)
        rows, radii = torch.stack(rows), torch.stack(radii)
    torch.cuda.synchronize()
    n = lambda t, like: (t if t is not None else torch.zeros_like(like)).double().cpu().numpy()  # noqa: E731
    return dict(grads={k: n(leaves[k].grad, leaves[k]) for k in B.RAW}, verts=n(verts.grad, verts),
                face=[n(t.grad, t) for t in (fc, fR, fs)], m2d=rows.double().cpu().numpy(),
                radii=radii.cpu().numpy())


def _check_backward(case, K, mode="exact"):
    bound = _case(case)["bound"]
    _, table = _rig(bound, K)
    gc, ga, gd = _upstream(bound, K)
    what = f"{case[0]} K={K} {mode}"
    got = _step(bound, table, gc, ga, gd, True, mode)
    ref = _step(bound, table, gc, ga, gd, False)
    for k in B.RAW:
        h.assert_grad_tight(got["grads"][k], ref["grads"][k], f"{what} d{k}", **STRICT)
    for name, a, b in zip(("face_center", "face_orien_mat", "face_scaling"), got["face"], ref["face"]):
        h.assert_grad_tight(a, b, f"{what} d{name}", **STRICT)
    h.assert_grad_tight(got["verts"], ref["verts"], f"{what} dverts", **STRICT)
    for k in range(K):
        h.assert_grad_tight(got["m2d"][k], ref["m2d"][k], f"{what} dmeans2D view {k}", **STRICT)
    dark = (got["radii"] == 0).all(0)
    for k in B.RAW:
        assert not got["grads"][k][dark].any(), f"{what}: d{k} nonzero for a splat culled in every view"
    assert not got["m2d"][got["radii"] == 0].any(), f"{what}: a dL/dmeans2D row nonzero where the radius is 0"
    return got, ref


@pytest.mark.parametrize("K", [2, 3, 6])
@pytest.mark.parametrize("name", ["near_plane", "saturating_stack", "guard_band+sh3", "faint", "tile_borders+ties"])
def test_backward_is_the_sum_of_single_view_depth_alpha_backwards(name, K):
    _check_backward((name, None, None), K)


@pytest.mark.parametrize("mode", ["late", "none"])
def test_backward_under_the_other_sync_modes(mode):
    _check_backward(("near_plane", None, None), 4, mode)


def test_backward_at_1080p_with_long_tile_lists():
    """The backward of two 1920x1080 views of an avatar scene against the two single-view backwards."""
    from tests.test_gpu_camera_fov import _rig as orbit_rig
    from gaussianavatars_b200.renderer import camera_table
    sc = h.avatar_scene(P=100_000, W=1920, H=1080, seed=8)
    bound = dict(params=sc["params"], verts=sc["verts"], faces=sc["faces"], bg=sc["bg"], W=1920, H=1080,
                 sh_degree=3)
    table = camera_table(orbit_rig(1920, 1080, n=4)[1:3], DEV)
    gc, ga, gd = _upstream(bound, 2)
    got = _step(bound, table, gc, ga, gd, True)
    ref = _step(bound, table, gc, ga, gd, False)
    for k in B.RAW:
        h.assert_grad_tight(got["grads"][k], ref["grads"][k], f"1080p d{k}")
    h.assert_grad_tight(got["verts"], ref["verts"], "1080p dverts")
    for k in range(2):
        h.assert_grad_tight(got["m2d"][k], ref["m2d"][k], f"1080p dmeans2D view {k}")


# ---- 3. gab200_backward_views on a depth-alpha state ----------------------------------------------------------------
def test_plain_backward_views_on_a_depth_alpha_state_is_the_colour_backward(monkeypatch):
    """gab200_backward_views (not gab200_backward_views_depth_alpha) on the state a K-view depth-alpha forward kept,
    against the plain K-view frame's backward.  The blend backward's atomics reorder float sums between any two runs,
    so the comparison is the strict gate, not bit equality."""
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound_views_train
    bound = _case(("guard_band+sh3", None, None))["bound"]
    K = 6
    _, table = _rig(bound, K)
    gc = _upstream(bound, K)[0]
    L = N.lib()
    plain_backward = L.gab200_backward_views
    calls = []

    def colour_only(b, views, cams, ga, gd, stream):
        calls.append(b._obj.state.contents.depth_prefix)
        return plain_backward(b, views, cams, stream)

    def step(depth_alpha):
        leaves, verts = _leaves(bound)
        fc, fR, fs = face_frame(verts, bound["faces"].to(DEV))
        m2d = torch.zeros((K, leaves["_xyz"].shape[0], 3), device=DEV, requires_grad=True)
        out = rasterize_bound_views_train(_settings(bound), table, *(leaves[n] for n in B.RAW),
                                          bound["params"]["binding"].to(DEV), fc, fR, fs, means2D=m2d,
                                          depth_alpha=depth_alpha)
        (out[0] * gc).sum().backward()
        torch.cuda.synchronize()
        return [leaves[n].grad for n in B.RAW] + [verts.grad, m2d.grad]

    monkeypatch.setattr(L, "gab200_backward_views_depth_alpha", colour_only)
    da = step(True)
    monkeypatch.undo()
    assert calls == [1], "the depth-alpha state was not handed to gab200_backward_views"
    plain = step(False)
    for i, (a, b) in enumerate(zip(da, plain)):
        h.assert_grad_tight(a.double().cpu().numpy(), b.double().cpu().numpy(), f"colour only [{i}]", **STRICT)


# ---- 4. against float64 at ragged sizes -----------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(15, 17), (33, 31), (4, 20)])
@pytest.mark.parametrize("name", ["near_plane", "saturating_stack", "faint", "tile_borders"])
def test_planes_and_summed_gradients_against_float64_at_ragged_sizes(name, W, H):
    from tests import planes64 as P64
    case = (name, W, H)
    c = _case(case)
    bound, cams = c["bound"], c["cams"]
    K = 6
    table = B.table(cams, DEV)
    gc, ga, gd = _upstream(bound, K, seed=11)
    got = _step(bound, table, gc, ga, gd, True)
    with torch.no_grad():
        from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound_views
        leaves, verts = _leaves(bound)
        frame = face_frame(verts.detach(), bound["faces"].to(DEV))
        _, _, _, _, alpha, depth = rasterize_bound_views(_settings(bound), table,
                                                         *(leaves[n].detach() for n in B.RAW),
                                                         bound["params"]["binding"].to(DEV), *frame,
                                                         display=False, float_image=True, depth_alpha=True)
    act32 = c["act"]
    d = torch.float64
    act, lv, vv = B.activate(bound, d, requires_grad=True)
    pinned = {k: v + (torch.as_tensor(e).to(d).reshape(v.shape) - v).detach()
              for (k, v), e in zip(((k, act[k]) for k in ("means3D", "opacities", "cov3D")),
                                   (act32[0], act32[1], act32[3]))}
    P = lv["_xyz"].shape[0]
    total = torch.zeros((), dtype=d)
    m2ds = []
    for k in range(K):
        m2 = torch.zeros(P, 3, dtype=d, requires_grad=True)
        m2ds.append(m2)
        st = c["sts"][k]
        if st is None:
            assert not alpha[k].any() and not depth[k].any()
            continue
        cam = cams[k]
        a_o, d_o, _ = P64.oracle_planes(act32[0].numpy(), act32[1].numpy(), cam, W, H, cov3D_precomp=act32[3].numpy())
        h.assert_image_close(alpha[k].cpu().numpy(), a_o, f"{name} {W}x{H} view {k}: alpha vs oracle")
        ds = max(1.0, float(abs(d_o).max()))
        h.assert_image_close(depth[k].cpu().numpy() / ds, d_o / ds, f"{name} {W}x{H} view {k}: depth vs oracle")
        pin = T.pin_of(st)
        idx = torch.nonzero(torch.from_numpy(pin["radii"]) > 0).reshape(-1)
        if idx.numel() == 0:
            continue
        img, a64, d64, _ = P64.render(pinned["means3D"][idx], m2[idx], pinned["opacities"][idx],
                                      cam.world_view_transform.to(d), cam.full_proj_transform.to(d),
                                      cam.camera_center.to(d), W, H, cam.tanfovx, cam.tanfovy, bound["bg"].to(d),
                                      shs=act["shs"][idx], sh_degree=bound["sh_degree"],
                                      cov3D_precomp=pinned["cov3D"][idx],
                                      radii=torch.from_numpy(pin["radii"]).long()[idx],
                                      rect_xy=torch.from_numpy(pin["xy"])[idx],
                                      depths=torch.from_numpy(pin["depths"])[idx])
        total = total + (img * gc[k].cpu().to(d)).sum() + (a64 * ga[k].cpu().to(d)).sum() + \
            (d64 * gd[k].cpu().to(d)).sum()
    leaf_list = [lv[k] for k in B.RAW] + [vv] + m2ds
    g64 = torch.autograd.grad(total, leaf_list, allow_unused=True)
    z = lambda t, like: (t if t is not None else torch.zeros_like(like)).detach().numpy()  # noqa: E731
    raw = {k: z(t, lv[k]) for k, t in zip(B.RAW, g64[:6])}
    rows = [None if c["sts"][k] is None else z(g64[7 + k], m2ds[k]) for k in range(K)]
    slack = {k: 0.0 for k in list(B.RAW) + ["verts"]}   # no fallback: the fixed gates only
    kes = [None if st is None else A.knife_edges(st) for st in c["sts"][:K]]
    _gate_all(f"{name}-{W}x{H} K={K} planes vs float64", got, raw, z(g64[6], vv), rows, K, slack, kes)


# ---- 5. FLAME -------------------------------------------------------------------------------------------------------
def test_plane_gradients_of_a_k_view_frame_reach_the_flame_parameters():
    """render_views_train(depth_alpha=True) with a mask and a depth term on a FLAME-posed head: the gradients of the
    posed FLAME rows equal the sum of the K single-view render(depth_alpha=True) steps."""
    from gaussianavatars_b200.renderer import render, render_views_train
    from tests import flame_oracle as fo
    from tests.test_gpu_camera_fov import _rig as orbit_rig
    from tests.test_gpu_train_step import _model
    sc = T.scene(P=1500, W=64, H=48)
    t, W, H, K = 2, sc["W"], sc["H"], 3
    cams = orbit_rig(W, H, n=K)
    bg = torch.ones(3, device=DEV)
    gen = torch.Generator().manual_seed(4)
    ga, gd = torch.randn((K, 1, H, W), generator=gen).to(DEV), torch.randn((K, 1, H, W), generator=gen).to(DEV)
    pc = _model(sc, 3)
    pc.select_mesh_by_timestep(t)
    out = render_views_train(cams, pc, Pipe, bg, depth_alpha=True)
    assert out["alpha"].shape == out["depth"].shape == (K, 1, H, W)
    ((out["alpha"] * ga).sum() + (out["depth"] * gd).sum()).backward()
    torch.cuda.synchronize()
    lib = {k: pc.flame_param[k].grad[t].double().cpu() for k in fo.POSED}
    ref = {k: torch.zeros_like(v) for k, v in lib.items()}
    for k, cam in enumerate(cams):
        pk = _model(sc, 3)
        pk.select_mesh_by_timestep(t)
        o = render(cam.to(DEV), pk, Pipe, bg, depth_alpha=True)
        assert torch.equal(o["alpha"], out["alpha"][k]) and torch.equal(o["depth"], out["depth"][k])
        ((o["alpha"] * ga[k]).sum() + (o["depth"] * gd[k]).sum()).backward()
        torch.cuda.synchronize()
        for n in fo.POSED:
            ref[n] += pk.flame_param[n].grad[t].double().cpu()
    for n in fo.POSED:
        h.assert_grad_tight(lib[n].numpy(), ref[n].numpy(), f"flame {n}")
    assert any(float(lib[n].abs().max()) > 0 for n in fo.POSED), "no plane gradient reached FLAME"
