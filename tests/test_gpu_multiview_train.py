"""-m gpu: the K cameras of one timestep as one training frame (gab200_forward_views_train, gab200_backward_views,
rasterize_bound_views_train, render_views_train).

The forward must equal gab200_forward_views and K single-camera forwards bit for bit (torch.equal).  The backward is
the sum over the views of the single-camera backward, formed in another order: it is compared with K single-camera
steps of this library, summed by autograd, under the tight elementwise gradient gate.  The densification statistics
of one K-view frame, fed row by row, must equal those of the K single-camera frames in view order."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import helpers as h
from tests.test_gpu_camera_fov import _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LEAVES = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")


@pytest.fixture(autouse=True)
def default_policies():
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    prev = R._EXACT_BINNING
    knob = N.tune(N.TUNE_TILE_SORT)
    yield
    R.set_exact_binning(prev)
    N.tune(N.TUNE_TILE_SORT, knob)
    R.set_sync_policy("late")
    R._capture_slot = None


def _table(cams, bad_fov=()):
    from gaussianavatars_b200.renderer import camera_table
    t = camera_table(cams, DEV)
    for k in bad_fov:
        t[k, 35] = 0.0
    return t.contiguous()


def _leaves(sc):
    p = sc["params"]
    leaves = {k: p[k].to(DEV).clone().requires_grad_(True) for k in LEAVES}
    verts = sc["verts"].to(DEV).clone().requires_grad_(True)
    return leaves, verts


def _settings(sc, row=None):
    from gaussianavatars_b200.rasterizer import GaussianRasterizationSettings
    bg = sc["bg"].to(DEV)
    if row is None:
        return GaussianRasterizationSettings(sc["H"], sc["W"], 1.0, 1.0, bg, 1.0, None, None, sc["sh_degree"], None,
                                             False, False)
    return GaussianRasterizationSettings(sc["H"], sc["W"], 1.0, 1.0, bg, 1.0, row[:16].clone(), row[16:32].clone(),
                                         sc["sh_degree"], row[32:35].clone(), False, False)


def _views_step(sc, table, dpix, hints=None):
    """One K-view training frame with dL/dimage = dpix: (color, radii, visibility, grads, verts.grad, means2D.grad)."""
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound_views_train, visible_of
    leaves, verts = _leaves(sc)
    fc, fR, fs = face_frame(verts, sc["faces"].to(DEV))
    K, P = table.shape[0], leaves["_xyz"].shape[0]
    m2d = torch.zeros((K, P, 3), device=DEV, requires_grad=True)
    sink = SimpleNamespace()
    color, radii = rasterize_bound_views_train(_settings(sc), table, *(leaves[k] for k in LEAVES),
                                               sc["params"]["binding"].to(DEV), fc, fR, fs, means2D=m2d,
                                               grad_sink=sink, hints=hints)
    vis = visible_of(radii).clone()
    (color * dpix).sum().backward()
    torch.cuda.synchronize()
    return color.detach(), radii, vis, {k: leaves[k].grad for k in LEAVES}, verts.grad, m2d.grad, sink


def _single_steps(sc, table, dpix):
    """K single-camera frames of the same leaves, one backward through the sum of their losses."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound, visible_of
    leaves, verts = _leaves(sc)
    fc, fR, fs = face_frame(verts, sc["faces"].to(DEV))
    K, P = table.shape[0], leaves["_xyz"].shape[0]
    R.set_sync_policy("exact")
    colors, radii, vis, m2ds, loss = [], [], [], [], 0.0
    for k in range(K):
        row = table[k]
        m2d = torch.zeros((P, 3), device=DEV, requires_grad=True)
        c, r = rasterize_bound(_settings(sc, row), *(leaves[n] for n in LEAVES), sc["params"]["binding"].to(DEV),
                               fc, fR, fs, means2D=m2d, tanfov=row[35:37].clone())
        vis.append(visible_of(r).clone())
        colors.append(c.detach())
        radii.append(r)
        m2ds.append(m2d)
        loss = loss + (c * dpix[k]).sum()
    loss.backward()
    torch.cuda.synchronize()
    R.set_sync_policy("late")
    return (torch.stack(colors), torch.stack(radii), torch.stack(vis), {k: leaves[k].grad for k in LEAVES},
            verts.grad, torch.stack([m.grad for m in m2ds]))


def _views_forward_only(sc, table):
    from gaussianavatars_b200.rasterizer import rasterize_bound_views, face_frame
    p = sc["params"]
    with torch.no_grad():
        fc, fR, fs = face_frame(sc["verts"].to(DEV), sc["faces"].to(DEV))
        color, _, radii, vis = rasterize_bound_views(_settings(sc), table, *(p[k].to(DEV) for k in LEAVES),
                                                     p["binding"].to(DEV), fc, fR, fs, display=False, float_image=True)
    return color, radii, vis


def _dpix(K, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((K, 3, H, W), generator=g) * 1e-3).to(DEV)


def _check_grads(views, singles, K, P):
    _, _, _, g_v, gv_v, m_v = views[:6]
    _, _, _, g_s, gv_s, m_s = singles
    for k in LEAVES:
        h.assert_grad_tight(g_v[k].cpu().numpy(), g_s[k].cpu().numpy(), f"d{k} (K={K})")
    h.assert_grad_tight(gv_v.cpu().numpy(), gv_s.cpu().numpy(), f"dverts (K={K})")
    for k in range(K):
        h.assert_grad_tight(m_v[k].cpu().numpy(), m_s[k].cpu().numpy(), f"dmeans2D view {k}")


@pytest.mark.parametrize("exact_binning", [False, True])
@pytest.mark.parametrize("tile_sort", [0, 1])
def test_training_forward_equals_forward_views_and_single_views_in_every_mode(exact_binning, tile_sort):
    """EXACT (no hint), LATE with a capacity far too small, NONE with room and NONE overflowing (sticky flag)."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    R.set_exact_binning(exact_binning)
    N.tune(N.TUNE_TILE_SORT, tile_sort)
    sc = h.avatar_scene(P=12_000, W=301, H=211, seed=4)
    table = _table(_rig(301, 211, n=3), bad_fov=(1,))
    K, P = 3, 12_000
    dpix = _dpix(K, 211, 301)
    singles = _single_steps(sc, table, dpix)
    fwd = _views_forward_only(sc, table)
    hints = R.FrameHints()
    exact = _views_step(sc, table, dpix, hints)
    n = hints.last["num_rendered"]
    assert hints.last["sync_mode"] == N.SYNC_EXACT and n > 0
    key = (DEV, 301, 211, P, K)
    hints.shapes[key] = (1024, (0, 0))
    late = _views_step(sc, table, dpix, hints)
    assert hints.last["sync_mode"] == N.SYNC_LATE and hints.last["attempts"] == 2
    runs = [exact, late]
    for cap in (n + 64, n // 4):
        R._capture_slot = R.CaptureSlot(DEV, cap)
        try:
            runs.append(_views_step(sc, table, dpix))
            flag = int(R._capture_slot.flag.item())
        finally:
            R._capture_slot = None
        assert flag == (0 if cap > n else 1)
    for r in runs[:3]:
        for got, want in ((r[0], singles[0]), (r[1], singles[1]), (r[2], singles[2])):
            assert torch.equal(got, want)
        assert torch.equal(r[0], fwd[0]) and torch.equal(r[1], fwd[1]) and torch.equal(r[2], fwd[2])
        _check_grads(r, singles, K, P)
    assert not singles[1][1].any() and not (runs[0][5][1] != 0).any()   # the invalid-FoV view: culled, no gradient


@pytest.mark.parametrize("K", [1, 3, 5])
def test_k_view_gradients_equal_the_sum_of_single_view_steps(K):
    sc = h.avatar_scene(P=20_000, W=480, H=352, seed=1, timestep=4)
    table = _table(_rig(480, 352, n=max(K, 2))[:K])
    dpix = _dpix(K, 352, 480, seed=K)
    views = _views_step(sc, table, dpix)
    singles = _single_steps(sc, table, dpix)
    assert torch.equal(views[0], singles[0]) and torch.equal(views[1], singles[1])
    _check_grads(views, singles, K, 20_000)
    flat = views[6].flat_grad
    assert flat.numel() == 20_000 * 59 and torch.equal(flat[:20_000 * 3].view(-1, 3), views[3]["_xyz"])


def test_four_views_at_1080p_with_long_tile_lists():
    """1920x1080, 100k splats plus 3000 copies of one splat: tile lists beyond 2048 entries in every view."""
    import gaussianavatars_b200.rasterizer as R
    sc = h.avatar_scene(P=100_000, W=1920, H=1080, seed=4)
    p = sc["params"]
    for k in p:
        p[k] = torch.cat([p[k], p[k][:1].expand(3000, *p[k].shape[1:])]).contiguous()
    P = p["_xyz"].shape[0]
    table = _table(_rig(1920, 1080, n=4))
    dpix = _dpix(4, 1080, 1920, seed=9)
    R.keep_last_state(True)
    try:
        singles = _single_steps(sc, table[:1], dpix[:1])
        _, _, ranges, _ = R.export_last_binning()
    finally:
        R.keep_last_state(False)
    assert int((ranges[:, 1] - ranges[:, 0]).max()) > 2048, "no tile list beyond the shared-memory sort"
    singles = _single_steps(sc, table, dpix)
    views = _views_step(sc, table, dpix)
    assert torch.equal(views[0], singles[0]) and torch.equal(views[1], singles[1])
    _check_grads(views, singles, 4, P)


def test_densification_statistics_equal_k_single_view_frames_in_order():
    from gaussianavatars_b200.densify import add_densification_stats
    sc = h.avatar_scene(P=20_000, W=320, H=240, seed=2)
    K, P = 4, 20_000
    table = _table(_rig(320, 240, n=K))
    dpix = _dpix(K, 240, 320, seed=3)
    views = _views_step(sc, table, dpix)
    singles = _single_steps(sc, table, dpix)

    def stats(m2d_rows, radii_rows):
        model = SimpleNamespace(xyz_gradient_accum=torch.zeros((P, 1), device=DEV),
                                denom=torch.zeros((P, 1), device=DEV), max_radii2D=torch.zeros((P,), device=DEV))
        for k in range(K):
            add_densification_stats(model, SimpleNamespace(grad=m2d_rows[k].contiguous()), radii_rows[k].contiguous())
        torch.cuda.synchronize()
        return model

    a, b = stats(views[5], views[1]), stats(singles[5], singles[1])
    assert torch.equal(a.denom, b.denom) and torch.equal(a.max_radii2D, b.max_radii2D)
    assert int(a.denom.max()) == K
    h.assert_grad_tight(a.xyz_gradient_accum.cpu().numpy(), b.xyz_gradient_accum.cpu().numpy(), "xyz_gradient_accum")


def test_render_views_train_returns_render_dicts_with_a_leading_k():
    """render_views_train against K render() calls: images and radii bit for bit; every raw-parameter gradient, the
    face-frame gradients and each view's viewspace_points.grad row under the tight gradient gate."""
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render, render_views_train
    sc = h.avatar_scene(P=8_000, W=256, H=192, seed=5)
    cams = [c for c in _rig(256, 192, n=3)]
    pipe = SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
    bg = sc["bg"].to(DEV)

    def model():
        pc = MeshBoundGaussians(sc["params"], 3, sc["verts"], sc["faces"], pose_fn=syn.pose_mesh, device=DEV,
                                requires_grad=True)
        pc.select_mesh_by_timestep(0)   # the face frame as leaves: its gradients land in .grad
        for n in ("face_center", "face_orien_mat", "face_scaling"):
            setattr(pc, n, getattr(pc, n).detach().clone().requires_grad_(True))
        return pc
    pc = model()
    out = render_views_train(cams, pc, pipe, bg)
    assert out["render"].shape == (3, 3, 192, 256) and out["radii"].shape == (3, 8_000)
    assert out["viewspace_points"].shape == (3, 8_000, 3)
    assert torch.equal(out["visibility_filter"], out["radii"] > 0)
    dpix = _dpix(3, 192, 256, seed=11)
    (out["render"] * dpix).sum().backward()
    pc1 = model()
    total, vps = 0.0, []
    for k, cam in enumerate(cams):
        o = render(cam, pc1, pipe, bg)
        assert torch.equal(o["render"], out["render"][k].detach()) and torch.equal(o["radii"], out["radii"][k])
        total = total + (o["render"] * dpix[k]).sum()
        vps.append(o["viewspace_points"])
    total.backward()
    for n in LEAVES:
        h.assert_grad_tight(getattr(pc, n).grad.cpu().numpy(), getattr(pc1, n).grad.cpu().numpy(), f"d{n}")
    for n in ("face_center", "face_orien_mat", "face_scaling"):
        h.assert_grad_tight(getattr(pc, n).grad.cpu().numpy(), getattr(pc1, n).grad.cpu().numpy(), f"d{n}")
    for k in range(3):
        h.assert_grad_tight(out["viewspace_points"].grad[k].cpu().numpy(), vps[k].grad.cpu().numpy(),
                            f"viewspace_points row {k}")


# ---- the float64 step ---------------------------------------------------------------------------------------------
def _oracle_cams(sc, K):
    """K cameras around the oracle scene's head (synthetic.look_at_camera from orbit poses), distinct FoVs."""
    import math
    from gaussianavatars_b200 import synthetic as syn
    cams = []
    for i in range(K):
        orb = syn.orbit_camera(sc["W"], sc["H"], r=1.0, fovy_deg=20.0, azimuth_deg=15.0 - 20.0 * i,
                               elevation_deg=4.0 * math.sin(i))
        f = 1.0 + 0.05 * i
        cams.append(syn.look_at_camera(sc["W"], sc["H"], math.degrees(orb.FoVx) * f, math.degrees(orb.FoVy) * f,
                                       w2c=orb.world_view_transform.T.numpy()))
    return cams


def _oracle_gts(sc, K):
    g = torch.Generator().manual_seed(31)
    return [sc["gt"]] + [torch.randint(0, 256, sc["gt"].shape, generator=g, dtype=torch.uint8) for _ in range(K - 1)]


def _eager_views_step(sc, t, fl, cams, gts):
    """The eager K-view step on the device: K x the batch photometric loss plus the regularisers of every view."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.renderer import render_views_train
    from tests.test_gpu_train_step import ATTR, _model, _n
    from tests import flame_oracle as fo
    from tests import train_step_oracle as T
    K = len(cams)
    pc = _model(sc, fl["sh_degree"])
    pc.select_mesh_by_timestep(t)
    pc.verts.retain_grad()
    out = render_views_train(cams, pc, SimpleNamespace(debug=False), torch.tensor(fl["bg"], device=DEV))
    photo = g.photometric_loss(out["render"], torch.stack(gts).to(DEV), fl["lambda_dssim"]) * float(K)
    lxs, lss = [], []
    for k in range(K):
        lx, ls = g.binding_regularizers(pc._xyz, pc._scaling, out["radii"][k], pc.binding, pc.face_scaling,
                                        **T.reg_kwargs(fl))
        lxs.append(lx)
        lss.append(ls)
    total = photo + sum(lxs) + sum(lss)
    total.backward()
    torch.cuda.synchronize()
    with torch.no_grad():
        act = g.bind_activate(1.0, pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc.binding, pc.face_center,
                              pc.face_orien_mat, pc.face_scaling)
    res = dict(parts=dict(xyz=float(sum(lxs).detach()), scale=float(sum(lss).detach()), total=float(total.detach())),
               grads={**{k: _n(getattr(pc, k).grad) for k in ATTR}, "verts": _n(pc.verts.grad)},
               flame={k: _n(pc.flame_param[k].grad) for k in fo.POSED},
               means2D=_n(out["viewspace_points"].grad), radii=out["radii"].cpu().numpy())
    shs = torch.cat((pc._features_dc, pc._features_rest), dim=1).detach()
    return res, act, shs


def _summed_references(sc, t, fl, cams, gts, act, shs):
    """Per camera: the C oracle's forward on the exported activation, the float64 step pinned to it and the float32
    reference step; and the sums over the cameras of both steps."""
    from tests import flame_oracle as fo
    from tests import train_step_oracle as T
    means3D, opac, scales, cov = act
    sts, r64s, r32s = [], [], []
    for cam, gt in zip(cams, gts):
        st = T.oracle_forward_on(means3D, opac, cam, sc["W"], sc["H"], fl, shs, cov3D=cov)
        args = (sc["params"], sc["flame_param"], t, sc["assets"], cam, gt, fl)
        sts.append(st)
        r64s.append(T.step(*args, torch.float64, pin=T.pin_of(st)))
        r32s.append(T.step(*args, torch.float32))

    def total(rs):
        out = dict(parts={k: sum(r["parts"][k] for r in rs) for k in ("xyz", "scale", "total")},
                   grads={k: sum(np.asarray(r["grads"][k], np.float64) for r in rs) for k in rs[0]["grads"]
                          if k != "means2D"},
                   flame={k: sum(np.asarray(r["flame"][k], np.float64) for r in rs) for k in fo.POSED})
        out["grads"]["means2D"] = None
        return out
    return sts, r64s, r32s, total(r64s), total(r32s)


def _gate_sum(title, got, s64, s32, t):
    """train_step_oracle's gates on the summed step.  A loss, vertex or FLAME record the fixed gate rejects passes
    only if its error stays within twice the SUMMED float32 reference's (the rule of test_gpu_train_step)."""
    from tests import train_step_oracle as T
    from tests.test_gpu_train_step import _array
    got = dict(got, grads={k: v for k, v in got["grads"].items() if k != "means2D"})
    ref = dict(s64, grads={k: v for k, v in s64["grads"].items() if v is not None})
    bad = []
    for r in T.gates(got, ref, t):
        print(f"[train-views] {title:<34s} {r['what']:<20s} worst={r['worst']:.2e} outliers={r['outliers']}/{r['allowed']}")
        if r["ok"]:
            continue
        if r["what"] in ("xyz", "scale", "total"):
            e_c, e_32 = abs(got["parts"][r["what"]] - s64["parts"][r["what"]]), \
                abs(s32["parts"][r["what"]] - s64["parts"][r["what"]])
        else:
            a = _array(got, r["what"], t)
            if a is None or "not zero" in r["what"]:
                bad.append(r["what"])
                continue
            ref64 = _array(s64, r["what"], t)
            e_c = float(np.abs(np.asarray(a, np.float64) - ref64).max())
            e_32 = float(np.abs(np.asarray(_array(s32, r["what"], t), np.float64) - ref64).max())
        print(f"[train-views] {title:<34s} {r['what']:<20s} beyond the fixed gate: {e_c:.3e}, 2 x fp32 {2 * e_32:.3e}")
        if e_c > 2 * e_32:
            bad.append(r["what"])
    assert not bad, f"{title}: fails {bad}"


@pytest.mark.parametrize("K", [1, 3, 5])
@pytest.mark.parametrize("scene", [0, 1])
def test_k_view_step_matches_the_sum_of_float64_steps(K, scene):
    """The eager K-view step (photometric loss, regularisers on each view's radii, FLAME timestep, face gradients)
    against the sum over the cameras of train_step_oracle.step in float64, each pinned to its own camera's decisions;
    each camera's dL/dmeans2D row against that camera's own float64 step."""
    from tests import train_step_oracle as T
    from tests.test_gpu_train_step import SCENES, _flags, _scene
    t, sh, metric = SCENES[scene]
    sc = _scene()
    fl = _flags(sc, sh, metric)
    cams, gts = _oracle_cams(sc, K), _oracle_gts(sc, K)
    got, act, shs = _eager_views_step(sc, t, fl, cams, gts)
    sts, r64s, _, s64, s32 = _summed_references(sc, t, fl, cams, gts, act, shs)
    for k in range(K):
        assert np.array_equal(got["radii"][k], sts[k].radii), f"view {k}: radii differ from the C oracle"
        rec = T.gate_splat(f"dL/dmeans2D view {k}", got["means2D"][k], r64s[k]["grads"]["means2D"])
        print(f"[train-views] means2D view {k}: worst={rec['worst']:.2e} outliers={rec['outliers']}/{rec['allowed']}")
        assert rec["ok"], f"view {k}: dL/dmeans2D fails its gate"
    _gate_sum(f"K={K} t={t} sh={sh} metric={metric}", got, s64, s32, t)


def test_atomic_face_reduction_of_the_views_backward_matches_the_float64_sum(monkeypatch):
    """The per-face gradients of gab200_backward_views summed by per-splat atomics (no CSR chunks given) pass the same
    gates and agree with the CSR route."""
    from gaussianavatars_b200 import rasterizer as R
    from tests import flame_oracle as fo
    from tests.test_gpu_train_step import SCENES, _flags, _scene
    t, sh, metric = SCENES[0]
    sc = _scene()
    fl = _flags(sc, sh, metric)
    cams, gts = _oracle_cams(sc, 3), _oracle_gts(sc, 3)
    csr, act, shs = _eager_views_step(sc, t, fl, cams, gts)
    real = R._face_csr
    monkeypatch.setattr(R, "_face_csr", lambda binding, F, chunk=16: (real(binding, F, chunk)[0], None))
    atomic, _, _ = _eager_views_step(sc, t, fl, cams, gts)
    _, _, _, s64, s32 = _summed_references(sc, t, fl, cams, gts, act, shs)
    _gate_sum("atomic K=3", atomic, s64, s32, t)
    a, c = atomic["grads"]["verts"], csr["grads"]["verts"]
    assert np.abs(a - c).max() <= 1e-5 * np.abs(c).max(), "dL/dverts: atomic and CSR routes differ"
    for k in fo.POSED:
        a, c = atomic["flame"][k], csr["flame"][k]
        assert np.abs(a - c).max() <= 1e-5 * np.abs(c).max(), f"dL/d{k}: atomic and CSR routes differ"


# ---- the K-view training replay -----------------------------------------------------------------------------------
W_G, H_G = 320, 240


def _flame_trainable():
    import gaussianavatars_b200 as g
    from tests.test_gpu_flame import LRS, _flame_model, _full_size, _lbs
    a, fp = _full_size(T=6, seed=2)
    pc = _flame_model(a, fp, _lbs(a))
    groups = [{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pc.parameters())]
    opt = g.Adam(groups + g.flame_param_groups(pc.flame_param), lr=0.0, eps=1e-15, capturable=True)
    P = pc._xyz.shape[0]
    for n in ("xyz_gradient_accum", "denom"):
        setattr(pc, n, torch.zeros((P, 1), device=DEV))
    pc.max_radii2D = torch.zeros((P,), device=DEV)
    return pc, opt


def _eager_k_iteration(pc, opt, t, cams, gt):
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.renderer import render_views_train
    opt.zero_grad(set_to_none=True)
    pc.select_mesh_by_timestep(t)
    out = render_views_train(cams, pc, SimpleNamespace(debug=False), torch.ones(3, device=DEV))
    loss = g.photometric_loss(out["render"], gt, 0.2) * float(len(cams))
    for k in range(len(cams)):
        lx, ls = g.binding_regularizers(pc._xyz, pc._scaling, out["radii"][k], pc.binding, pc.face_scaling)
        loss = loss + lx + ls
    loss.backward()
    vp = out["viewspace_points"].grad
    for k in range(len(cams)):
        g.add_densification_stats(pc, SimpleNamespace(grad=vp[k]), out["radii"][k])
    opt.step()
    torch.cuda.synchronize()
    return float(loss.detach()), out["render"].detach()


def test_k_view_graphed_frame_matches_eager_k_view_iterations_without_recapture():
    """Capturable Adam over the splat and FLAME groups, the FLAME head and densify_stats in one K = 3 replay per
    iteration, against the same iterations run eagerly; new cameras, timesteps and ground truth never re-capture, and
    after_backward sees the flat gradient buffer summed over the views."""
    from gaussianavatars_b200.graph import GraphedFrame
    from tests.test_gpu_flame import LRS
    pc, opt = _flame_trainable()
    pe, opt_e = _flame_trainable()
    P = pc._xyz.shape[0]
    rig = [c.to(DEV) for c in _rig(W_G, H_G, n=6)]
    groups = [rig[:3], rig[3:]]
    seen = []
    fr = GraphedFrame(pc, W_G, H_G, 1.0, 1.0, torch.ones(3), loss="photometric", regularizers={}, optimizer=opt,
                      densify_stats=True, views_per_replay=3, warm_cameras=groups,
                      after_backward=lambda: seen.append(pc.flat_grad))
    gen = torch.Generator().manual_seed(3)
    steps = [(0, 0), (1, 1), (2, 0), (3, 1), (1, 0)]
    for i, (t, gi) in enumerate(steps):
        gt = torch.randint(0, 256, (3, 3, H_G, W_G), generator=gen, dtype=torch.uint8).to(DEV)
        fr.set_inputs(cameras=groups[gi], timestep=t, gt_u8=gt)
        fr.run(check=True)
        torch.cuda.synchronize()
        loss, img = _eager_k_iteration(pe, opt_e, t, groups[gi], gt)
        if i == 0:   # later steps start from parameters that differ by the summation order of earlier gradients
            assert torch.equal(fr.image, img), "the first replay's images differ from the eager iteration's"
        rel = abs(float(fr.loss) - loss) / abs(loss)
        print(f"[k-graph] step {i} t={t} loss graph {float(fr.loss):.7f} eager {loss:.7f} rel {rel:.1e}")
        assert rel <= 1e-4, f"step {i}: loss differs"
    assert fr.captures == 1 and not fr.overflowed()
    assert seen and seen[-1] is fr.flat_grad and fr.flat_grad.numel() == P * 59
    for n, p, q in zip(LRS, pc.parameters(), pe.parameters()):
        d = (p.detach() - q.detach()).abs()
        bound = 2 * len(steps) * LRS[n]
        frac = float((d > 0.25 * bound).float().mean())
        print(f"[k-graph] {n:<9s} max|diff| {float(d.max()):.2e} (Adam bound {bound:.1e}) frac>bound/4 {frac:.1e}")
        assert frac <= 1e-2, n
    for n in ("denom", "max_radii2D"):
        assert float((getattr(pc, n) != getattr(pe, n)).float().mean()) <= 1e-3, n
    assert int(pc.denom.max()) > 3   # the views of several iterations were counted
    a, b = pc.xyz_gradient_accum, pe.xyz_gradient_accum
    assert float(((a - b).abs() > 1e-3 * b.abs() + 1e-6 * float(b.abs().max())).float().mean()) <= 1e-2
    assert float(opt.state[pc._xyz]["step"]) == len(steps)


def test_k_view_graphed_frame_overflow_applies_no_step_and_check_recovers():
    from gaussianavatars_b200.graph import GraphedFrame
    pc, opt = _flame_trainable()
    rig = [c.to(DEV) for c in _rig(W_G, H_G, n=3)]
    fr = GraphedFrame(pc, W_G, H_G, 1.0, 1.0, torch.ones(3), loss="l1_u8", optimizer=opt, densify_stats=True,
                      views_per_replay=3, capacity=2048)
    gt = torch.full((3, 3, H_G, W_G), 128, dtype=torch.uint8, device=DEV)
    fr.set_inputs(cameras=rig, timestep=1, gt_u8=gt)
    before = [p.detach().clone() for p in pc.parameters()]
    fr.run()
    assert fr.overflowed(), "a 2048-instance capacity must overflow three views"
    for p, q in zip(pc.parameters(), before):
        assert torch.equal(p.detach(), q), "an overflowed replay changed a parameter"
    assert int(pc.denom.max()) == 0 and float(opt.state[pc._xyz]["step"]) == 0
    fr.run(check=True)
    assert not fr.overflowed() and fr.captures == 2
    assert float(opt.state[pc._xyz]["step"]) == 1 and int(pc.denom.max()) == 3


def test_k_view_graphed_frame_with_host_inputs():
    """host_inputs: a host (K, 37) table and a host (K,3,H,W) ground truth are uploaded on the copy stream; the loss
    of the replay equals the eager K-view loss."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.graph import GraphedFrame
    from gaussianavatars_b200.renderer import camera_table, render_views_train
    pc, _ = _flame_trainable()
    rig = [c.to(DEV) for c in _rig(W_G, H_G, n=2)]
    fr = GraphedFrame(pc, W_G, H_G, 1.0, 1.0, torch.ones(3), loss="l1_u8", host_inputs=True, views_per_replay=2,
                      warm_cameras=[rig])
    table = camera_table(rig, DEV).cpu()
    gt = torch.randint(0, 256, (2, 3, H_G, W_G), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    fr.set_inputs(cameras=table, gt_u8=gt, timestep=2)
    fr.run(check=True)
    torch.cuda.synchronize()
    pc.select_mesh_by_timestep(2)
    with torch.no_grad():
        out = render_views_train(rig, pc, SimpleNamespace(debug=False), torch.ones(3, device=DEV))
        ref = float(g.l1_loss_u8(out["render"], gt.to(DEV))) * 2
    assert torch.equal(fr.image, out["render"])
    assert abs(float(fr.loss_host) - ref) <= 1e-6 * ref
