"""-m gpu: the field of view read from device memory (gab200_forward_device_fov / gab200_backward_device_fov,
rasterize_bound(tanfov=), GraphedFrame(per_camera_fov=True)) against the host-float path with the same float values,
one captured graph over a rig of cameras with distinct fields of view, and the culled result of an invalid value.

Images, radii and visibility are compared bit for bit.  Gradients are compared at the atomic-summation-order tolerance
of the other graph tests: the blend backward and the face-frame backward sum with floating-point atomics, so two runs
of the SAME host-float path may already differ in the last bits."""
import math
from dataclasses import replace
from types import SimpleNamespace

import pytest
import torch

from tests import helpers as h

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def _grads_close(a, b, what, rtol=2e-5):
    for k, (x, y) in enumerate(zip(a, b)):
        if y is None:
            assert x is None, what
            continue
        scale = float(y.abs().max()) + 1e-30
        d = float((x - y).abs().max())
        assert d <= rtol * scale, f"{what}: gradient {k} differs by {d:.3e} (max|ref| {scale:.3e})"


def _cam_with_fov(cam, fov_deg):
    """The camera's pose with another field of view ('orbit' keeps the orbit camera's own)."""
    from gaussianavatars_b200 import synthetic as syn
    if fov_deg == "orbit":
        return cam
    return syn.look_at_camera(cam.image_width, cam.image_height, fov_deg, fov_deg,
                              w2c=cam.world_view_transform.T.numpy())


def _dev_tanfov(cam):
    from gaussianavatars_b200.graph import tanfov_floats
    return tanfov_floats(cam.FoVx, cam.FoVy).to(DEV)


class _Sync:
    """Runs a call under one of the three sync modes; LATE with a capacity far too small, so that the re-enqueue
    path runs too."""

    def __init__(self, mode, key):
        self.mode, self.key = mode, key
        self.hints = None

    def __call__(self, fn):
        import gaussianavatars_b200.rasterizer as R
        self.hints = R.FrameHints()
        R.set_sync_policy("exact" if self.mode == "exact" else "late")
        try:
            if self.mode == "late":
                self.hints.set_capacity(self.key, 1024)
                self.hints.set_depth(self.key, (0, 0))
            if self.mode == "none":
                R._capture_slot = R.CaptureSlot(DEV, 4_000_000)
            out = fn(self.hints)
        finally:
            R._capture_slot = None
            R.set_sync_policy("late")
        if self.mode == "late":
            assert R.last_frame_info()["attempts"] == 2 and R.last_frame_info()["sync_mode"] == 1
        return out


def _bound_run(sc, cam, tanfov, sync, seed=3):
    """Fused route with a trainable mesh: image, radii, visibility, splat gradients, face-frame gradients, dL/dverts."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound
    p = sc["params"]
    leaves = [p[k].to(DEV).clone().requires_grad_(True)
              for k in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")]
    verts = sc["verts"].to(DEV).clone().requires_grad_(True)
    fc, fR, fs = face_frame(verts, sc["faces"].to(DEV))
    for t in (fc, fR, fs):
        t.retain_grad()
    rs = h.cuda_settings(dict(cam=cam, W=sc["W"], H=sc["H"], bg=sc["bg"], sh_degree=3), DEV, debug=False)
    m2 = torch.zeros((leaves[0].shape[0], 3), device=DEV, requires_grad=True)

    def go(hints):
        sink = SimpleNamespace(_gab200_hints=hints)
        return rasterize_bound(rs, *leaves, binding=p["binding"].to(DEV), face_center=fc, face_orien_mat=fR,
                               face_scaling=fs, means2D=m2, grad_sink=sink, tanfov=tanfov)
    img, radii = sync(go)
    vis = R.visible_of(radii).clone()
    gout = torch.randn(img.shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
    (img * gout).sum().backward()
    torch.cuda.synchronize()
    grads = [x.grad for x in leaves] + [m2.grad, fc.grad, fR.grad, fs.grad, verts.grad]
    return img.detach(), radii, vis, grads


def _activated_run(sc, cam, tanfov, sync, seed=3):
    """Reference surface (ACTIVATED inputs) through the C ABI directly."""
    import ctypes as C
    from gaussianavatars_b200 import _native as N
    import gaussianavatars_b200.rasterizer as R
    P = sc["means3D"].shape[0]
    t = {k: sc[k].to(DEV).contiguous() for k in ("means3D", "opacities", "scales", "rotations", "shs")}
    rs = h.cuda_settings(dict(cam=cam, W=sc["W"], H=sc["H"], bg=sc["bg"], sh_degree=sc["sh_degree"]), DEV, debug=False)
    a = N.ForwardArgs()
    keep = R._fill_common(a, rs, DEV, P, True)
    a.input_mode = N.INPUT_ACTIVATED
    a.sh_coeffs = t["shs"].shape[1]
    a.means3D, a.opacities, a.scales, a.rotations, a.shs = (t[k].data_ptr() for k in
                                                             ("means3D", "opacities", "scales", "rotations", "shs"))
    img, radii, st, holder = sync(lambda hints: R._run_forward(a, DEV, True, hints, tanfov))
    vis = R.visible_of(radii).clone()
    gout = torch.randn(img.shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
    e = lambda *s: torch.zeros(s, dtype=torch.float32, device=DEV)  # noqa: E731
    gr = dict(m3=e(P, 3), m2=e(P, 3), op=e(P, 1), col=e(P, 3), sh=e(*t["shs"].shape), sc=e(P, 3), rot=e(P, 4), cov=e(P, 6))
    b = N.BackwardArgs()
    b.abi_version = N.ABI_VERSION
    b.fwd, b.state = C.pointer(a), C.pointer(st)
    b.dL_dout_color = gout.data_ptr()
    b.dL_dmeans3D, b.dL_dmeans2D, b.dL_dopacity = gr["m3"].data_ptr(), gr["m2"].data_ptr(), gr["op"].data_ptr()
    b.dL_dcolors, b.dL_dshs = gr["col"].data_ptr(), gr["sh"].data_ptr()
    b.dL_dscales, b.dL_drotations, b.dL_dcov3D = gr["sc"].data_ptr(), gr["rot"].data_ptr(), gr["cov"].data_ptr()
    R._run_backward(b, DEV, tanfov)
    torch.cuda.synchronize()
    del keep, holder
    return img, radii, vis, list(gr.values())


def _scene(mode):
    if mode == "bound":
        return h.avatar_scene(P=12_000, W=320, H=240, seed=4)
    return h.random_scene(P=10_000, W=320, H=240, sh_degree=3, seed=4)   # its own camera stands for 'orbit'


@pytest.mark.parametrize("sync", ["exact", "late", "none"])
@pytest.mark.parametrize("fov", [20.0, "orbit", 90.0])
@pytest.mark.parametrize("mode", ["bound", "activated"])
def test_device_fov_equals_host_fov(mode, fov, sync):
    sc = _scene(mode)
    cam = _cam_with_fov(sc["cam"], fov)
    run = _bound_run if mode == "bound" else _activated_run
    P = (sc["params"]["_xyz"] if mode == "bound" else sc["means3D"]).shape[0]
    key = (DEV, sc["W"], sc["H"], P)
    ref = run(sc, cam, None, _Sync(sync, key))
    got = run(sc, cam, _dev_tanfov(cam), _Sync(sync, key))
    assert int((ref[1] > 0).sum()) > 100, "scene renders nothing"
    assert torch.equal(got[0], ref[0]), "image differs"
    assert torch.equal(got[1], ref[1]), "radii differ"
    assert torch.equal(got[2], ref[2]), "visibility differs"
    _grads_close(got[3], ref[3], f"{mode} fov={fov} sync={sync}")


def test_null_device_fov_is_the_existing_entry_point(monkeypatch):
    from gaussianavatars_b200 import _native as N
    sc = _scene("bound")
    key = (DEV, sc["W"], sc["H"], sc["params"]["_xyz"].shape[0])
    ref = _bound_run(sc, sc["cam"], None, _Sync("exact", key))
    L = N.lib()
    fwd, bwd = L.gab200_forward_device_fov, L.gab200_backward_device_fov
    monkeypatch.setattr(L, "gab200_forward", lambda a, st, s: fwd(a, None, st, s))
    monkeypatch.setattr(L, "gab200_backward", lambda b, s: bwd(b, None, s))
    got = _bound_run(sc, sc["cam"], None, _Sync("exact", key))
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2])
    _grads_close(got[3], ref[3], "NULL tanfov")


@pytest.mark.parametrize("tanfov", [(0.0, 0.0), (0.3, 0.0), (-0.5, 0.4), (float("nan"), float("nan")),
                                    (float("inf"), 0.3)])
def test_invalid_device_fov_culls_every_splat(tanfov):
    sc = _scene("bound")
    key = (DEV, sc["W"], sc["H"], sc["params"]["_xyz"].shape[0])
    t = torch.tensor(tanfov, dtype=torch.float32, device=DEV)
    img, radii, vis, grads = _bound_run(sc, sc["cam"], t, _Sync("exact", key))
    assert int(radii.abs().sum()) == 0 and not bool(vis.any())
    bg = sc["bg"].to(DEV).view(3, 1, 1).expand_as(img)
    assert torch.equal(img, bg), "an invalid field of view must render the background"
    for g in grads:
        assert bool(torch.isfinite(g).all()) and float(g.abs().max()) == 0.0


# ---- one graph over a rig ---------------------------------------------------------------------------------------
def _rig(W, H, n=16, base_fovy=20.0, spread=0.08):
    """n cameras around the head with distinct poses and fields of view (base x (1 -+ spread))."""
    from gaussianavatars_b200 import synthetic as syn
    cams = []
    for i in range(n):
        orb = syn.orbit_camera(W, H, r=1.0, fovy_deg=base_fovy, azimuth_deg=-50 + 100 * i / (n - 1),
                               elevation_deg=6 * math.sin(i))
        f = 1.0 + spread * (2 * i / (n - 1) - 1)
        cams.append(syn.look_at_camera(W, H, math.degrees(orb.FoVx) * f, math.degrees(orb.FoVy) * f,
                                       w2c=orb.world_view_transform.T.numpy()))
    return cams


def _bound_model(sc):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    return MeshBoundGaussians(sc["params"], 3, sc["verts"], sc["faces"], pose_fn=syn.pose_mesh, device=DEV,
                              requires_grad=True)


def _eager(sc, cam, gt):
    """Eager render() (host field of view) + the photometric loss + backward on a fresh model."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.renderer import render
    pc = _bound_model(sc)
    v = sc["verts"].to(DEV).clone().requires_grad_(True)
    pc.update_mesh_properties(v)
    out = render(cam.to(DEV), pc, Pipe, sc["bg"].to(DEV))
    g.photometric_loss(out["render"], gt, 0.2).backward()
    torch.cuda.synchronize()
    return out["render"].detach(), [p.grad for p in pc.parameters()] + [v.grad]


def test_one_graph_renders_every_camera_of_a_rig_with_its_own_fov():
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    sc = h.avatar_scene(P=15_000, W=400, H=304, seed=5)
    cams = _rig(sc["W"], sc["H"])
    assert len({(c.FoVx, c.FoVy) for c in cams}) == 16
    gt = torch.randint(0, 256, (3, sc["H"], sc["W"]), generator=torch.Generator().manual_seed(7),
                       dtype=torch.uint8).to(DEV)
    pc = _bound_model(sc)
    blocks = [camera_block(c, fov=True).to(DEV) for c in cams]
    fr = GraphedFrame(pc, sc["W"], sc["H"], cams[0].FoVx, cams[0].FoVy, sc["bg"], loss="photometric",
                      warm_cameras=blocks, per_camera_fov=True)
    fr.set_inputs(camera=blocks[0], verts=sc["verts"].to(DEV), gt_u8=gt)
    for i in list(range(16)) + [3, 0]:
        fr.set_inputs(camera=cams[i])
        fr.run(check=True)
        torch.cuda.synchronize()
        img, grads = _eager(sc, cams[i], gt)
        assert torch.equal(fr.image, img), f"camera {i}: replay differs from the eager render()"
        _grads_close([p.grad for p in pc.parameters()] + [fr.verts.grad], grads, f"camera {i}")
    assert fr.captures == 1 and not fr.overflowed()

    # only the two field-of-view floats change: the replay must follow them
    cam = cams[5]
    wide = replace(cam, FoVx=cam.FoVx * 1.3, FoVy=cam.FoVy * 1.3)
    fr.set_inputs(camera=cam)
    fr.run(check=True)
    before = fr.image.clone()
    blk = camera_block(cam, fov=True)
    blk[35:] = camera_block(wide, fov=True)[35:]
    assert torch.equal(blk[:35], camera_block(wide)[:35])
    fr.set_inputs(camera=blk.to(DEV))
    fr.run(check=True)
    torch.cuda.synchronize()
    assert not torch.equal(fr.image, before), "changing the device field of view changed nothing"
    img, _ = _eager(sc, wide, gt)
    assert torch.equal(fr.image, img), "replay at the new field of view differs from the eager render()"
    assert fr.captures == 1


def test_warm_up_sizes_the_capacity_with_each_cameras_own_fov():
    """A zoomed-in camera of the rig needs more instances than the others: the warm-up renders it with its own field
    of view, so no replay over the rig overflows."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    from gaussianavatars_b200.renderer import render
    sc = h.avatar_scene(P=15_000, W=400, H=304, seed=6)
    cams = _rig(sc["W"], sc["H"], n=6, spread=0.0)
    cams[4] = replace(_rig(sc["W"], sc["H"], n=6, base_fovy=12.0)[4])   # narrow: larger on screen
    need = []
    pc_e = _bound_model(sc)
    pc_e.update_mesh_properties(sc["verts"].to(DEV))
    hints = R.hints_of(pc_e)
    with torch.no_grad():
        for c in cams:
            render(c.to(DEV), pc_e, Pipe, sc["bg"].to(DEV))
            need.append(hints.last["num_rendered"])
    assert need[4] > max(need[:4] + need[5:]), need
    pc = _bound_model(sc)
    blocks = [camera_block(c, fov=True).to(DEV) for c in cams]
    fr = GraphedFrame(pc, sc["W"], sc["H"], cams[0].FoVx, cams[0].FoVy, sc["bg"], loss="dL_dimage",
                      warm_cameras=blocks, per_camera_fov=True, headroom=1.0)
    fr.set_inputs(camera=blocks[0], verts=sc["verts"].to(DEV))
    fr.capture()
    assert fr.slot.capacity >= need[4]
    for b in blocks:
        fr.set_inputs(camera=b)
        fr.run(check=False)
    assert not fr.overflowed(wait=True) and fr.captures == 1


def test_full_training_iteration_over_a_rig_with_distinct_fovs():
    """8 iterations of the full graph (capturable Adam over the splat and FLAME groups, densification statistics,
    regularisers, the FLAME head posed inside) over cameras with distinct fields of view, against the eager
    iteration; the tolerances of the FLAME full-iteration test."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    from gaussianavatars_b200.renderer import render
    from tests import flame_oracle as fo
    from tests.test_gpu_flame import ASSET_KEYS, LRS, W_IMG, H_IMG, _flame_model, _full_size, _lbs
    a, fp = _full_size(T=6, seed=2)
    cams = _rig(W_IMG, H_IMG, n=8)
    gt = torch.randint(0, 256, (3, H_IMG, W_IMG), generator=torch.Generator().manual_seed(7), dtype=torch.uint8).to(DEV)
    pc = _flame_model(a, fp, _lbs(a))
    opt = g.Adam([{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pc.parameters())] +
                 g.flame_param_groups(pc.flame_param), lr=0.0, eps=1e-15, capturable=True)
    P = pc._xyz.shape[0]
    for m in (pc,):
        m.xyz_gradient_accum, m.denom = torch.zeros((P, 1), device=DEV), torch.zeros((P, 1), device=DEV)
        m.max_radii2D = torch.zeros((P,), device=DEV)
    blocks = [camera_block(c, fov=True).to(DEV) for c in cams]
    fr = GraphedFrame(pc, W_IMG, H_IMG, cams[0].FoVx, cams[0].FoVy, torch.ones(3), loss="photometric",
                      regularizers={}, optimizer=opt, densify_stats=True, warm_cameras=blocks, per_camera_fov=True)
    fr.set_inputs(camera=blocks[0], gt_u8=gt, timestep=0)

    pe = _flame_model(a, fp, _lbs(a))
    oa = fo.assets_as({k: a[k] for k in (*ASSET_KEYS, "parents")}, torch.float32, DEV)
    opt_s = g.Adam([{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pe.parameters())], lr=0.0, eps=1e-15)
    opt_f = torch.optim.Adam(g.flame_param_groups(pe.flame_param), lr=0.0, eps=1e-15)
    pe.xyz_gradient_accum, pe.denom = torch.zeros((P, 1), device=DEV), torch.zeros((P, 1), device=DEV)
    pe.max_radii2D = torch.zeros((P,), device=DEV)
    f0 = {k: pe.flame_param[k].detach().clone() for k in fo.POSED}
    steps = [0, 1, 2, 3, 1, 0, 2, 3]
    for i, t in enumerate(steps):
        fr.set_inputs(camera=blocks[i], timestep=t)
        fr.run(check=True)
        opt_s.zero_grad(set_to_none=True)
        opt_f.zero_grad(set_to_none=True)
        verts, _, _ = fo.select_mesh_by_timestep(oa, pe.flame_param, t)
        pe.update_mesh_properties(verts[0])
        out = render(cams[i].to(DEV), pe, Pipe, torch.ones(3, device=DEV))
        loss = g.photometric_loss(out["render"], gt, 0.2)
        lx, ls = g.binding_regularizers(pe._xyz, pe._scaling, out["radii"], pe.binding, pe.face_scaling)
        (loss + lx + ls).backward()
        g.add_densification_stats(pe, SimpleNamespace(grad=out["viewspace_points"].grad), out["radii"])
        opt_s.step()
        opt_f.step()
        torch.cuda.synchronize()
        rel = abs(float(fr.loss) - float(loss + lx + ls)) / abs(float(loss + lx + ls))
        print(f"[fov-train] step {i} camera FoVy {math.degrees(cams[i].FoVy):.2f} deg loss rel diff {rel:.1e}")
        assert rel <= 1e-4, f"step {i}: loss differs"
    assert fr.captures == 1 and not fr.overflowed()
    for k in fo.POSED:
        dg = (pc.flame_param[k].detach() - f0[k]).cpu()
        de = (pe.flame_param[k].detach() - f0[k]).cpu()
        assert torch.count_nonzero(dg[4:]) == 0 and torch.count_nonzero(de[4:]) == 0, "unvisited rows moved"
        err = float((dg - de).abs().max()) / (float(de.abs().max()) + 1e-30)
        assert err <= 0.05, k
    for n, p, q in zip(LRS, pc.parameters(), pe.parameters()):
        d = (p.detach() - q.detach()).abs()
        frac = float((d > 0.25 * 2 * len(steps) * LRS[n]).float().mean())
        assert frac <= 1e-2, n
    for n in ("denom", "max_radii2D"):
        assert torch.equal(getattr(pc, n), getattr(pe, n)) or \
            float((getattr(pc, n) != getattr(pe, n)).float().mean()) <= 1e-3, n
    assert float(opt.state[pc.flame_param["expr"]]["step"]) == len(steps)
