"""-m gpu: the capture's RGBA frames as the ground truth of the captured training iteration.

  * gab200_composite_rgba / composite_rgba against the reference loader's own bytes for every (colour, alpha) pair
    (tests/golden/rgba_composite_vectors.npz), and against the float64-then-truncate restatement the CPU tests prove
    equal to the loader, at ragged sizes, on offset slices, for other background colours and for K = 16 at 550x802;
  * GraphedFrame(rgba=True) against GraphedFrame fed composite_rgba's bytes, for K = 1 and K = 4;
  * GraphedFrame(rgba=True, lambda_mask=0.1) against the eager iteration (composite_rgba -> render(depth_alpha=True)
    -> loss + mask term -> backward -> statistics -> capturable Adam), and its loss against a float64 restatement;
  * host inputs through a prefetching pair, and an overflowing replay that applies no step.

Replays and their references start every iteration from the same state.  Images, alpha planes, ground truth, masks,
radii and the visibility counts are compared with torch.equal; the gradients differ only by the order of the
backward's atomic sums and are held to the gate of the other graph tests.  For K = 1 the step is also checked
bit for bit: the parameters, moments and statistics after a replay equal the eager statistics + Adam step applied to
the replay's own gradients."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import test_gpu_train_graph as TG
from tests import test_gpu_multiview_train as MV
from tests.test_gpu_camera_fov import _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "rgba_composite_vectors.npz"))
LAM = 0.1


def _g():
    import gaussianavatars_b200 as g
    return g


def composite64(rgba: np.ndarray, bg) -> np.ndarray:
    """The loader's arithmetic in numpy's order, float64, then truncation: (..., H, W, 4) -> (..., 3, H, W)."""
    norm = rgba / 255.0
    arr = norm[..., :3] * norm[..., 3:4] + np.asarray(bg, dtype=np.float64) * (1 - norm[..., 3:4])
    return np.moveaxis(np.trunc(arr * 255.0).astype(np.uint8), -1, -3)


def _rgba(K, H, W, seed):
    """(K, H, W, 4) uint8 host frames: random colours, an opaque ellipse, transparent outside, random alpha between."""
    gen = torch.Generator().manual_seed(seed)
    rgba = torch.randint(0, 256, (K, H, W, 4), generator=gen, dtype=torch.uint8)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    r = (xx / 0.55) ** 2 + (yy / 0.75) ** 2
    a = rgba[..., 3]
    a[:, r < 0.8] = 255
    a[:, r > 1.3] = 0
    return rgba


# ---- the kernel ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,bg", [("bg0", 0.0), ("bg1", 1.0)])
def test_composite_equals_the_loader_bytes_for_every_pair(name, bg):
    g = _g()
    rgba = torch.from_numpy(GOLD["rgba"]).to(DEV)
    gt, mask = g.composite_rgba(rgba, torch.full((3,), bg))
    want = torch.from_numpy(GOLD[name]).to(DEV)
    bad = int((gt != want).sum())
    print(f"[rgba] {name}: {bad} of {want.numel()} bytes differ from the loader")
    assert gt.shape == (3, 256, 256) and mask.shape == (1, 256, 256)
    assert torch.equal(gt, want)
    assert torch.equal(mask[0], rgba[..., 3])
    # a batch of the frame over per-channel mixed backgrounds: channel ch takes its background's bytes
    mixed = torch.tensor([bg, 1.0 - bg, bg])
    gt2, mask2 = g.composite_rgba(torch.stack([rgba, rgba]), mixed)
    other = torch.from_numpy(GOLD["bg1" if name == "bg0" else "bg0"]).to(DEV)
    for k in range(2):
        assert torch.equal(gt2[k, 0], want[0]) and torch.equal(gt2[k, 1], other[1]) and torch.equal(gt2[k, 2], want[2])
        assert torch.equal(mask2[k, 0], rgba[..., 3])


@pytest.mark.parametrize("K,H,W", [(1, 37, 29), (3, 37, 29), (2, 32, 32), (3, 5, 7), (1, 1, 1), (16, 550, 802)])
@pytest.mark.parametrize("bg", [(0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.25, 0.6, 0.9)])
def test_composite_matches_the_float64_restatement(K, H, W, bg):
    g = _g()
    rgba = _rgba(K, H, W, seed=K * 1000 + H)
    want = composite64(rgba.numpy(), np.asarray(bg, dtype=np.float32).astype(np.float64))
    gt, mask = g.composite_rgba(rgba.to(DEV), torch.tensor(bg))
    assert torch.equal(gt.cpu(), torch.from_numpy(want))
    assert torch.equal(mask.cpu()[:, 0], rgba[..., 3])
    if K == 1:   # the (H, W, 4) form of one frame
        gt1, mask1 = g.composite_rgba(rgba[0].to(DEV), torch.tensor(bg))
        assert gt1.shape == (3, H, W) and torch.equal(gt1, gt[0]) and torch.equal(mask1, mask[0])


@pytest.mark.parametrize("shift", [1, 16, 4])
def test_composite_on_offset_slices(shift):
    """Inputs and outputs that are views at a byte offset into a larger buffer (the scalar path for 1, the vector path
    for 16-byte input / 4-byte output offsets when H*W % 4 == 0), and a NULL mask."""
    from gaussianavatars_b200.training import launch_composite_rgba
    K, H, W = 3, 24, 20
    rgba = _rgba(K, H, W, seed=shift)
    bg = torch.tensor([1.0, 0.0, 1.0], device=DEV)
    want = torch.from_numpy(composite64(rgba.numpy(), [1.0, 0.0, 1.0]))
    src_buf = torch.zeros(rgba.numel() + shift, dtype=torch.uint8, device=DEV)
    src = src_buf[shift:].view(K, H, W, 4)
    src.copy_(rgba.to(DEV))
    out_shift = shift % 8 if shift != 16 else 4
    out_buf = torch.full((K * 3 * H * W + out_shift,), 7, dtype=torch.uint8, device=DEV)
    gt = out_buf[out_shift:].view(K, 3, H, W)
    mask_buf = torch.full((K * H * W + out_shift,), 7, dtype=torch.uint8, device=DEV)
    mask = mask_buf[out_shift:].view(K, 1, H, W)
    launch_composite_rgba(src, bg, gt, mask)
    assert torch.equal(gt.cpu(), want) and torch.equal(mask.cpu()[:, 0], rgba[..., 3])
    assert bool((out_buf[:out_shift] == 7).all()) and bool((mask_buf[:out_shift] == 7).all())
    gt.zero_()
    launch_composite_rgba(src[1:], bg, gt[1:], None)   # a view sliced out of the batch, no mask
    assert torch.equal(gt[1:].cpu(), want[1:]) and bool((gt[0] == 0).all())


# ---- the captured frame: shared helpers -------------------------------------------------------------------------
def _copy_state(dst, dopt, src, sopt):
    """dst's trained tensors, moments, step counters and statistics := src's, in place (no re-capture)."""
    dopt.init_state()
    sopt.init_state()
    with torch.no_grad():
        for gd, gs in zip(dopt.param_groups, sopt.param_groups):
            for p, q in zip(gd["params"], gs["params"]):
                p.copy_(q)
                for k, v in sopt.state.get(q, {}).items():
                    dopt.state[p][k].copy_(v)
        for n in TG.STATS:
            getattr(dst, n).copy_(getattr(src, n))


def _compare(what, image, ref_image, loss, ref_loss, pc, pc_ref, opt, opt_ref, alpha=None, ref_alpha=None):
    assert torch.equal(image, ref_image), f"{what}: image differs"
    if alpha is not None:
        assert torch.equal(alpha, ref_alpha), f"{what}: alpha plane differs"
    rel = abs(loss - ref_loss) / abs(ref_loss)
    print(f"[rgba] {what}: loss {loss:.8f} ref {ref_loss:.8f} rel {rel:.1e}")
    assert rel <= 1e-6, f"{what}: loss differs"
    TG._grads_close([p.grad for p in pc.parameters()], [p.grad for p in pc_ref.parameters()])
    assert torch.equal(pc.denom, pc_ref.denom) and torch.equal(pc.max_radii2D, pc_ref.max_radii2D), what
    for gr, gq in zip(opt.param_groups, opt_ref.param_groups):
        for p, q in zip(gr["params"], gq["params"]):
            assert torch.equal(opt.state[p]["step"], opt_ref.state[q]["step"]), what
            d = (p.detach() - q.detach()).abs()
            # Adam moves a parameter by at most ~lr per step: the two steps' gradients differ by summation order only
            assert float((d > 0.25 * gr["lr"] + 1e-7).float().mean()) <= 1e-2, f"{what}: {gr.get('name')}"


def _single_view_setup(seed=0):
    sc, _ = TG._scene()
    rgba = _rgba(1, sc["H"], sc["W"], seed)[0]
    return sc, rgba


def _single_frame(pc, sc, **kw):
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    cam = sc["cam"]
    fr = GraphedFrame(pc, sc["W"], sc["H"], cam.FoVx, cam.FoVy, sc["bg"], loss="photometric", regularizers={},
                      optimizer=pc.optimizer, densify_stats=True, **kw)
    fr.set_inputs(camera=camera_block(cam), verts=sc["verts"].to(DEV))
    return fr


def _check_step_exact(fr, pc, snap, what):
    """The replay's parameters, moments and statistics equal the eager statistics + Adam step on its own gradients."""
    grads = [p.grad for p in pc.parameters()]
    ps, opt, m = TG._expected_after_step(pc, snap, grads, fr.viewspace_points.grad, fr.radii)
    for p, q in zip(pc.parameters(), ps):
        assert torch.equal(p.detach(), q.detach()), f"{what}: parameter differs from the eager step"
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(pc.optimizer.state[p][k], opt.state[q][k]), f"{what}: {k} differs"
    for n in TG.STATS:
        assert torch.equal(getattr(pc, n), getattr(m, n)), f"{what}: {n} differs"


# ---- rgba=True, lambda_mask=0: the frame fed the composite's bytes -----------------------------------------------
@pytest.mark.parametrize("K", [1, 4])
def test_rgba_frame_equals_the_frame_fed_the_composite_bytes(K):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.graph import GraphedFrame
    g = _g()
    if K == 1:
        sc, _ = _single_view_setup()
        pa, pb = TG._trainable(sc), TG._trainable(sc)
        oa, ob = pa.optimizer, pb.optimizer
        fa, fb = _single_frame(pa, sc, rgba=True), _single_frame(pb, sc)
        bg, H, W = sc["bg"].to(DEV), sc["H"], sc["W"]
        poses = [sc["verts"], syn.pose_mesh(sc["verts"], 9), sc["verts"]]
        inputs = [dict(verts=v.to(DEV)) for v in poses]
    else:
        (pa, oa), (pb, ob) = MV._flame_trainable(), MV._flame_trainable()
        rig = [c.to(DEV) for c in _rig(MV.W_G, MV.H_G, n=8)]
        groups = [rig[:4], rig[4:]]
        kw = dict(loss="photometric", regularizers={}, densify_stats=True, views_per_replay=4, warm_cameras=groups)
        fa = GraphedFrame(pa, MV.W_G, MV.H_G, 1.0, 1.0, torch.ones(3), optimizer=oa, rgba=True, **kw)
        fb = GraphedFrame(pb, MV.W_G, MV.H_G, 1.0, 1.0, torch.ones(3), optimizer=ob, **kw)
        bg, H, W = torch.ones(3, device=DEV), MV.H_G, MV.W_G
        inputs = [dict(cameras=groups[0], timestep=0), dict(cameras=groups[1], timestep=3),
                  dict(cameras=groups[0], timestep=1)]
    for i, inp in enumerate(inputs):
        rgba = _rgba(K, H, W, seed=10 + i).to(DEV)
        rgba = rgba[0] if K == 1 else rgba
        gt, mask = g.composite_rgba(rgba, bg)
        _copy_state(pb, ob, pa, oa)
        snap = TG._snapshot(pa) if K == 1 else None
        fa.set_inputs(gt_rgba=rgba, **inp)
        fb.set_inputs(gt_u8=gt, **inp)
        fa.run(check=True)
        fb.run(check=True)
        torch.cuda.synchronize()
        assert torch.equal(fa.gt, gt) and torch.equal(fa.mask, mask), f"replay {i}: composite differs"
        assert fa.alpha is None and fa.depth is None
        _compare(f"K={K} replay {i}", fa.image, fb.image, float(fa.loss), float(fb.loss), pa, pb, oa, ob)
        assert torch.equal(fa.radii, fb.radii)
        if snap is not None:
            _check_step_exact(fa, pa, snap, f"replay {i}")
    assert fa.captures == 1 and fb.captures == 1


# ---- lambda_mask > 0: the eager iteration --------------------------------------------------------------------------
def _eager_mask_iteration_single(sc, snap, verts, rgba, active_sh_degree):
    """composite_rgba -> render(depth_alpha=True) -> photometric + mask term + regularisers -> backward, on a model
    holding the pre-replay parameters: (image, alpha, loss, model)."""
    from gaussianavatars_b200.renderer import render
    g = _g()
    pc_e = TG._model(sc)
    for attr, q in zip(TG.ATTR.values(), snap["params"]):
        setattr(pc_e, attr, q.clone().requires_grad_(True))
    pc_e.active_sh_degree = active_sh_degree
    pc_e.update_mesh_properties(verts.to(DEV).clone().requires_grad_(True))
    bg = sc["bg"].to(DEV)
    gt, mask = g.composite_rgba(rgba, bg)
    out = render(sc["cam"].to(DEV), pc_e, TG.Pipe, bg, depth_alpha=True)
    loss = g.photometric_loss(out["render"], gt, 0.2)
    loss = loss + g.l1_loss_u8(out["alpha"], mask) * (1.0 * LAM)
    lx, ls = g.binding_regularizers(pc_e._xyz, pc_e._scaling, out["radii"], pc_e.binding, pc_e.face_scaling)
    loss = loss + lx + ls
    loss.backward()
    torch.cuda.synchronize()
    return out["render"].detach(), out["alpha"].detach(), float(loss), pc_e


def test_mask_term_replays_equal_the_eager_iteration():
    from gaussianavatars_b200 import synthetic as syn
    sc, _ = _single_view_setup()
    pc = TG._trainable(sc)
    fr = _single_frame(pc, sc, rgba=True, lambda_mask=LAM)
    for i, verts in enumerate((sc["verts"], syn.pose_mesh(sc["verts"], 9), sc["verts"])):
        rgba = _rgba(1, sc["H"], sc["W"], seed=20 + i)[0].to(DEV)
        snap = TG._snapshot(pc)
        img, alpha, loss, pc_e = _eager_mask_iteration_single(sc, snap, verts, rgba, pc.active_sh_degree)
        fr.set_inputs(verts=verts.to(DEV), gt_rgba=rgba)
        fr.run(check=True)
        torch.cuda.synchronize()
        assert torch.equal(fr.image, img) and torch.equal(fr.alpha, alpha), f"replay {i}: planes differ"
        assert fr.alpha.shape == (1, sc["H"], sc["W"]) and fr.depth.shape == (1, sc["H"], sc["W"])
        rel = abs(float(fr.loss) - loss) / loss
        print(f"[rgba] mask replay {i}: loss {float(fr.loss):.8f} eager {loss:.8f} rel {rel:.1e}")
        assert rel <= 1e-6
        TG._grads_close([p.grad for p in pc.parameters()], [p.grad for p in pc_e.parameters()])
        _check_step_exact(fr, pc, snap, f"mask replay {i}")
    assert fr.captures == 1


def _eager_k_mask_iteration(pc, opt, t, cams, rgba):
    from gaussianavatars_b200.renderer import render_views_train
    g = _g()
    opt.zero_grad(set_to_none=True)
    pc.select_mesh_by_timestep(t)
    bg = torch.ones(3, device=DEV)
    gt, mask = g.composite_rgba(rgba, bg)
    K = len(cams)
    out = render_views_train(cams, pc, SimpleNamespace(debug=False), bg, depth_alpha=True)
    loss = g.l1_loss_u8(out["render"], gt) * float(K)
    loss = loss + g.l1_loss_u8(out["alpha"], mask) * (float(K) * LAM)
    loss.backward()
    vp = out["viewspace_points"].grad
    for k in range(K):
        g.add_densification_stats(pc, SimpleNamespace(grad=vp[k]), out["radii"][k])
    opt.step()
    torch.cuda.synchronize()
    return out["render"].detach(), out["alpha"].detach(), float(loss), gt, mask


def _loss64(image, alpha, rgba, bg, K):
    """K mean|image - gt/255| + K lambda mean|alpha - a/255| in float64, the ground truth restated on the host."""
    gt = composite64(rgba.cpu().numpy(), np.asarray(bg, dtype=np.float64)).astype(np.float64) / 255.0
    a = rgba.cpu().numpy()[..., 3].astype(np.float64) / 255.0
    img = image.cpu().numpy().astype(np.float64).reshape(gt.shape)
    al = alpha.cpu().numpy().astype(np.float64).reshape(a.shape)
    return K * np.abs(img - gt).mean() + K * LAM * np.abs(al - a).mean()


def test_k_view_mask_term_replays_equal_the_eager_k_view_iteration():
    from gaussianavatars_b200.graph import GraphedFrame
    K = 4
    (pc, opt), (pe, opt_e) = MV._flame_trainable(), MV._flame_trainable()
    rig = [c.to(DEV) for c in _rig(MV.W_G, MV.H_G, n=8)]
    groups = [rig[:4], rig[4:]]
    fr = GraphedFrame(pc, MV.W_G, MV.H_G, 1.0, 1.0, torch.ones(3), loss="l1_u8", optimizer=opt, densify_stats=True,
                      views_per_replay=K, warm_cameras=groups, rgba=True, lambda_mask=LAM)
    for i, (t, gi) in enumerate([(0, 0), (2, 1), (1, 0)]):
        rgba = _rgba(K, MV.H_G, MV.W_G, seed=30 + i).to(DEV)
        _copy_state(pe, opt_e, pc, opt)
        fr.set_inputs(cameras=groups[gi], timestep=t, gt_rgba=rgba)
        fr.run(check=True)
        torch.cuda.synchronize()
        img, alpha, loss, gt, mask = _eager_k_mask_iteration(pe, opt_e, t, groups[gi], rgba)
        assert torch.equal(fr.gt, gt) and torch.equal(fr.mask, mask)
        assert fr.alpha.shape == (K, 1, MV.H_G, MV.W_G) and fr.depth.shape == (K, 1, MV.H_G, MV.W_G)
        _compare(f"K-view mask replay {i}", fr.image, img, float(fr.loss), loss, pc, pe, opt, opt_e, fr.alpha, alpha)
        l64 = _loss64(fr.image, fr.alpha, rgba, [1.0, 1.0, 1.0], K)
        rel = abs(float(fr.loss) - l64) / l64
        print(f"[rgba] K-view replay {i}: loss {float(fr.loss):.8f} float64 {l64:.8f} rel {rel:.1e}")
        assert rel <= 1e-6
    assert fr.captures == 1


# ---- host inputs, overflow, refusals -----------------------------------------------------------------------------
def test_prefetching_pair_with_rgba_host_inputs():
    """Two frames with host_inputs prefetch each other's pinned RGBA frame and camera inside their graphs; each
    replay's ground truth, mask and loss are those of the frame that was staged for it."""
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    from gaussianavatars_b200.renderer import render
    from gaussianavatars_b200 import synthetic as syn
    g = _g()
    sc, _ = _single_view_setup()
    pc = TG._model(sc)
    cams = [sc["cam"], syn.orbit_camera(sc["W"], sc["H"], r=1.1, fovy_deg=22.0, azimuth_deg=-20.0)]
    frames = []
    for k in range(2):
        f = GraphedFrame(pc, sc["W"], sc["H"], sc["cam"].FoVx, sc["cam"].FoVy, sc["bg"], loss="l1_u8",
                         host_inputs=True, rgba=True, lambda_mask=LAM, per_camera_fov=True, warm_cameras=cams)
        assert f.gt_stage.shape == (sc["H"], sc["W"], 4) and f.gt_stage.is_pinned()
        f.set_inputs(verts=sc["verts"].to(DEV))
        frames.append(f)
    frames[0].prefetch_for(frames[1])
    frames[1].prefetch_for(frames[0])
    for f in frames:
        f.capture()
    rgbas = [_rgba(1, sc["H"], sc["W"], seed=40 + i)[0] for i in range(5)]
    frames[0].cam_stage.copy_(camera_block(cams[0], fov=True))
    frames[0].gt_stage.copy_(rgbas[0])
    frames[0].upload_staged()
    bg = sc["bg"].to(DEV)
    for i in range(5):
        cur, nxt = frames[i % 2], frames[(i + 1) % 2]
        torch.cuda.synchronize()
        if i + 1 < 5:
            nxt.cam_stage.copy_(camera_block(cams[(i + 1) % 2], fov=True))
            nxt.gt_stage.copy_(rgbas[i + 1])
        cur.run(check=True)
        torch.cuda.synchronize()
        gt, mask = g.composite_rgba(rgbas[i].to(DEV), bg)
        assert torch.equal(cur.gt, gt) and torch.equal(cur.mask, mask), f"step {i}: composite differs"
        pc.update_mesh_properties(sc["verts"].to(DEV))
        out = render(cams[i % 2].to(DEV), pc, TG.Pipe, bg, depth_alpha=True)
        ref = float(g.l1_loss_u8(out["render"], gt)) + float(g.l1_loss_u8(out["alpha"], mask)) * LAM
        assert torch.equal(cur.image, out["render"].detach()) and torch.equal(cur.alpha, out["alpha"].detach()), \
            f"step {i}"
        assert abs(float(cur.loss_host) - ref) <= 1e-6 * ref
        l64 = _loss64(cur.image, cur.alpha, rgbas[i], sc["bg"].numpy().astype(np.float32), 1)
        assert abs(float(cur.loss_host) - l64) <= 1e-6 * l64
    assert all(f.captures == 1 for f in frames)


def test_overflowing_mask_replay_applies_no_step_and_check_recovers():
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.graph import camera_block
    sc, _ = _single_view_setup()
    pc = TG._trainable(sc)
    other = syn.orbit_camera(sc["W"], sc["H"], r=1.0, fovy_deg=20.0, azimuth_deg=25.0)
    fr = _single_frame(pc, sc, rgba=True, lambda_mask=LAM, warm_cameras=[camera_block(sc["cam"]), camera_block(other)])
    rgba = _rgba(1, sc["H"], sc["W"], seed=50)[0].to(DEV)
    fr.set_inputs(gt_rgba=rgba)
    pc.optimizer.init_state()
    snap = TG._snapshot(pc)
    fr.capture(capacity=4096)
    fr.run(check=False)
    assert fr.overflowed(wait=True), "an overflowing replay was not flagged"
    TG._assert_state_equal(pc, snap, "overflowing replay")
    img, alpha, loss, pc_e = _eager_mask_iteration_single(sc, snap, sc["verts"], rgba, pc.active_sh_degree)
    fr.run(check=True)
    torch.cuda.synchronize()
    assert fr.captures == 2 and not fr.overflowed(wait=True)
    assert torch.equal(fr.image, img) and torch.equal(fr.alpha, alpha)
    assert abs(float(fr.loss) - loss) <= 1e-6 * loss
    TG._grads_close([p.grad for p in pc.parameters()], [p.grad for p in pc_e.parameters()])
    _check_step_exact(fr, pc, snap, "regrown replay")
    assert float(pc.optimizer.state[pc._xyz]["step"]) == 1.0


def test_rgba_frame_refusals():
    from gaussianavatars_b200.graph import GraphedFrame
    sc, _ = _single_view_setup()
    pc = TG._model(sc)
    kw = dict(loss="l1_u8")
    fr = GraphedFrame(pc, sc["W"], sc["H"], 1.0, 1.0, sc["bg"], rgba=True, **kw)
    plain = GraphedFrame(pc, sc["W"], sc["H"], 1.0, 1.0, sc["bg"], **kw)
    assert fr.gt_rgba.shape == (sc["H"], sc["W"], 4) and fr.mask.shape == (1, sc["H"], sc["W"])
    assert plain.gt_rgba is None and plain.mask is None and plain.lambda_mask == 0.0
    with pytest.raises(ValueError, match="give gt_rgba=, not gt_u8"):
        fr.set_inputs(gt_u8=torch.zeros(3, sc["H"], sc["W"], dtype=torch.uint8))
    with pytest.raises(ValueError, match="needs a frame built with rgba=True"):
        plain.set_inputs(gt_rgba=torch.zeros(sc["H"], sc["W"], 4, dtype=torch.uint8))
    for bad in (torch.zeros(sc["H"], sc["W"], 3, dtype=torch.uint8), torch.zeros(sc["H"], sc["W"], 4),
                torch.zeros(1, sc["H"], sc["W"], 4, dtype=torch.uint8)):
        with pytest.raises(ValueError, match="gt_rgba of this frame"):
            fr.set_inputs(gt_rgba=bad)
    ha = GraphedFrame(pc, sc["W"], sc["H"], 1.0, 1.0, sc["bg"], host_inputs=True, rgba=True, **kw)
    hb = GraphedFrame(pc, sc["W"], sc["H"], 1.0, 1.0, sc["bg"], host_inputs=True, **kw)
    with pytest.raises(ValueError, match="rgba=True on both"):
        ha.prefetch_for(hb)
    with pytest.raises(ValueError, match="rgba=True on both"):
        hb.prefetch_for(ha)
