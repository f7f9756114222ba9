"""-m gpu: the tile-packed lossless frame store (csrc/frames.cu, gaussianavatars_b200.frames.FrameStore) and the
captured training iteration that decodes its ground truth from it (GraphedFrame(frames=store)).

  * the device encoder writes the records and the index of oracle/frame_codec.py byte for byte;
  * the decode returns the frames it was given, bit for bit, for K = 1..16 ids (repeated, permuted, spanning several
    add() batches and an arena growth), with the mask plane written or not;
  * add_rgba is composite_rgba followed by add;
  * GraphedFrame(frames=store) against GraphedFrame(rgba=True) fed the same RGBA frames, K = 1, 4 and 16 at 550x802,
    with and without the mask term: gt and mask bytes, images, loss, gradients, parameters and Adam state, held to the
    standard of tests/test_gpu_rgba_mask.py;
  * a prefetching host-input pair, an overflowing replay that regrows, and re-capture only when the store grows."""
import numpy as np
import pytest
import torch

from oracle import frame_codec as fc
from tests import test_gpu_multiview_train as MV
from tests import test_gpu_rgba_mask as RM
from tests import test_gpu_train_graph as TG
from tests.test_gpu_camera_fov import _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LAM = 0.1
KINDS = ["noise", "constant", "ramp", "spike", "binary"]
SIZES = [(1, 1), (1, 17), (17, 1), (15, 16), (550, 802), (1080, 1920)]


def _g():
    import gaussianavatars_b200 as g
    return g


def _frames(kind, F, H, W, seed=0):
    from tests.test_oracle_frame_codec import _frames as make
    gt, mask = make(kind, F, H, W, seed)
    return torch.from_numpy(gt), torch.from_numpy(mask)


# ---- the codec on the device ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("H,W", SIZES)
def test_device_records_and_index_equal_the_oracle(kind, H, W):
    F = 2 if H * W <= 550 * 802 else 1
    gt, mask = _frames(kind, F, H, W, seed=H * 7 + W)
    store = _g().FrameStore(W, H, [1.0, 1.0, 1.0], DEV)
    assert store.add(gt.to(DEV), mask.to(DEV)) == list(range(F))
    arena, base, off = fc.encode_frames(gt.numpy(), mask.numpy())
    torch.cuda.synchronize()
    assert store.nbytes == arena.size + F * (8 + 4 * off.shape[1]) and store.raw_nbytes == F * 4 * H * W
    assert np.array_equal(store.frame_base[:F].cpu().numpy(), base)
    assert np.array_equal(store.tile_off[:F * off.shape[1]].cpu().numpy().view(np.uint32), off.reshape(-1))
    dev_arena = store.arena[:arena.size].cpu().numpy()
    bad = int((dev_arena != arena).sum())
    print(f"[frames] {kind} {H}x{W}: {arena.size} B for {F} frames ({store.nbytes / store.raw_nbytes:.3f} of raw), "
          f"{bad} bytes differ")
    assert bad == 0
    # no mask: M = 255
    s2 = _g().FrameStore(W, H, [1.0, 1.0, 1.0], DEV)
    s2.add(gt[0].to(DEV))
    a2, _, _ = fc.encode_frames(gt[:1].numpy(), None)
    assert np.array_equal(s2.arena[:a2.size].cpu().numpy(), a2)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("H,W", SIZES)
def test_decode_returns_the_frames_bit_for_bit(kind, H, W):
    F = 3 if H * W <= 550 * 802 else 2
    gt, mask = _frames(kind, F, H, W, seed=H + 3 * W)
    store = _g().FrameStore(W, H, [0.0, 0.0, 0.0], DEV)
    store.add(gt.to(DEV), mask.to(DEV))
    ids = [F - 1, 0, F - 1, 1 % F]
    g2, m2 = store.decode(ids)
    assert torch.equal(g2.cpu(), gt[ids]) and torch.equal(m2.cpu(), mask[ids])


def test_decode_k_1_to_16_across_batches_and_an_arena_growth():
    """Frames added in three batches (one without a mask) -- the arena and the index reallocate on the way -- then
    decoded K = 1..16 at a time with repeated and permuted ids; the mask plane written or left alone."""
    g = _g()
    H, W = 550, 802
    store = g.FrameStore(W, H, [1.0, 1.0, 1.0], DEV)
    parts = [_frames("binary", 3, H, W, seed=1), _frames("noise", 2, H, W, seed=2), _frames("ramp", 4, H, W, seed=3)]
    gts, masks, moved = [], [], 0
    for i, (gt, mask) in enumerate(parts):
        before = store.pointers()
        ids = store.add(gt.to(DEV), None if i == 1 else mask.to(DEV))
        done = sum(x.shape[0] for x in gts)
        assert ids == list(range(done, done + gt.shape[0]))
        moved += store.pointers()[0] != before[0]
        gts.append(gt)
        masks.append(torch.full_like(mask, 255) if i == 1 else mask)
    assert moved >= 2, "the arena did not grow across the batches"
    gt_all, mask_all = torch.cat(gts), torch.cat(masks)
    n = gt_all.shape[0]
    gen = torch.Generator().manual_seed(5)
    for K in range(1, 17):
        ids = torch.randint(0, n, (K,), generator=gen).tolist()
        g2, m2 = store.decode(ids)
        assert torch.equal(g2.cpu(), gt_all[ids]) and torch.equal(m2.cpu(), mask_all[ids]), f"K={K}"
    # the mask plane not written; a single (3,H,W) frame
    ids = torch.tensor([8, 0, 4], dtype=torch.int32, device=DEV)
    gt_out = torch.empty((3, 3, H, W), dtype=torch.uint8, device=DEV)
    store.launch_decode(ids, gt_out, None)
    assert torch.equal(gt_out.cpu(), gt_all[[8, 0, 4]])
    one = torch.empty((3, H, W), dtype=torch.uint8, device=DEV)
    one_mask = torch.empty((1, H, W), dtype=torch.uint8, device=DEV)
    store.launch_decode(ids[2:], one, one_mask)
    assert torch.equal(one.cpu(), gt_all[4]) and torch.equal(one_mask.cpu(), mask_all[4])
    # nbytes: noise costs its raw size plus the bounded overhead, the rest far less
    T = store.n_tiles
    assert store.nbytes <= n * fc.frame_bound(T)
    print(f"[frames] 9 frames at {W}x{H}: {store.nbytes} B, {store.raw_nbytes / store.nbytes:.2f}x smaller than raw")


def test_add_refusals_and_store_ids():
    g = _g()
    store = g.FrameStore(20, 10, [0.0, 0.0, 0.0], DEV)
    for bad in (torch.zeros(3, 10, 21, dtype=torch.uint8), torch.zeros(4, 10, 20, dtype=torch.uint8),
                torch.zeros(3, 10, 20), np.zeros((3, 10, 20), np.uint8)):
        with pytest.raises(ValueError, match="gt_u8 must be a uint8"):
            store.add(bad)
    with pytest.raises(ValueError, match="mask_u8 must be a uint8"):
        store.add(torch.zeros(3, 10, 20, dtype=torch.uint8), torch.zeros(3, 10, 20, dtype=torch.uint8))
    with pytest.raises(ValueError, match="mask_u8 holds 2 frames"):
        store.add(torch.zeros(1, 3, 10, 20, dtype=torch.uint8), torch.zeros(2, 1, 10, 20, dtype=torch.uint8))
    assert store.add(torch.zeros(0, 3, 10, 20, dtype=torch.uint8)) == [] and len(store) == 0
    assert store.add(torch.zeros(3, 10, 20, dtype=torch.uint8)) == [0]   # a host frame is uploaded
    with pytest.raises(ValueError, match="frame ids index the store's 1 frames"):
        store.decode([0, 1])


def test_add_rgba_is_composite_then_add():
    g = _g()
    H, W = 550, 802
    bg = [1.0, 0.0, 1.0]
    rgba = RM._rgba(3, H, W, seed=7)
    a = g.FrameStore(W, H, bg, DEV)
    b = g.FrameStore(W, H, bg, DEV)
    assert a.add_rgba(rgba) == [0, 1, 2]            # a host batch
    assert a.add_rgba(rgba[1].to(DEV)) == [3]       # one device frame
    gt, mask = g.composite_rgba(rgba.to(DEV), torch.tensor(bg))
    b.add(gt, mask)
    b.add(gt[1], mask[1])
    torch.cuda.synchronize()
    assert a._used == b._used and torch.equal(a.arena[:a._used], b.arena[:b._used])
    assert torch.equal(a.frame_base[:4], b.frame_base[:4]) and torch.equal(a.tile_off[:4 * a.n_tiles],
                                                                            b.tile_off[:4 * b.n_tiles])
    g2, m2 = a.decode([3, 0, 2])
    assert torch.equal(g2, gt[[1, 0, 2]]) and torch.equal(m2, mask[[1, 0, 2]])
    print(f"[frames] synthetic RGBA ellipse frames: {a.raw_nbytes / a.nbytes:.2f}x smaller than raw")


# ---- the captured iteration ----------------------------------------------------------------------------------------
H_S, W_S = 550, 802


def _pair_of_frames(K, lam, **kw):
    """Two FLAME models in the same state, a GraphedFrame(rgba=True) on one and a GraphedFrame(frames=store) on the
    other, over a rig of 550x802 cameras."""
    from gaussianavatars_b200.graph import GraphedFrame
    (pa, oa), (pb, ob) = MV._flame_trainable(), MV._flame_trainable()
    rig = [c.to(DEV) for c in _rig(W_S, H_S, n=max(2 * K, 2))]
    groups = [rig[:K], rig[K:2 * K]] if K > 1 else [rig[0], rig[1]]
    common = dict(loss="photometric", regularizers={}, densify_stats=True, views_per_replay=K, warm_cameras=groups,
                  per_camera_fov=True, lambda_mask=lam, **kw)
    bg = torch.ones(3)
    store = _g().FrameStore(W_S, H_S, bg, DEV)
    rgbas = RM._rgba(2 * K + 1, H_S, W_S, seed=K)
    store.add_rgba(rgbas)
    fa = GraphedFrame(pa, W_S, H_S, 1.0, 1.0, bg, optimizer=oa, rgba=True, **common)
    fb = GraphedFrame(pb, W_S, H_S, 1.0, 1.0, bg, optimizer=ob, frames=store, **common)
    return (pa, oa, fa), (pb, ob, fb), groups, store, rgbas


@pytest.mark.parametrize("lam", [0.0, LAM])
@pytest.mark.parametrize("K", [1, 4, 16])
def test_store_frame_equals_the_rgba_frame_fed_the_same_frames(K, lam):
    (pa, oa, fa), (pb, ob, fb), groups, store, rgbas = _pair_of_frames(K, lam)
    n = len(store)
    gen = torch.Generator().manual_seed(11 + K)
    for i, t in enumerate((0, 3, 1)):
        ids = torch.randint(0, n, (K,), generator=gen).tolist()
        ids[-1] = ids[0]   # a repeated frame
        cam = groups[i % 2]
        pose = dict(cameras=cam) if K > 1 else dict(camera=cam)
        RM._copy_state(pb, ob, pa, oa)
        fa.set_inputs(gt_rgba=(rgbas[ids] if K > 1 else rgbas[ids[0]]).to(DEV), timestep=t, **pose)
        fb.set_inputs(frames=ids if K > 1 else ids[0], timestep=t, **pose)
        fa.run(check=True)
        fb.run(check=True)
        torch.cuda.synchronize()
        assert torch.equal(fb.gt, fa.gt) and torch.equal(fb.mask, fa.mask), f"replay {i}: decoded bytes differ"
        assert torch.equal(fb.frame_ids.cpu(), torch.tensor(ids, dtype=torch.int32))
        RM._compare(f"store K={K} lam={lam} replay {i}", fb.image, fa.image, float(fb.loss), float(fa.loss), pb, pa,
                    ob, oa, fb.alpha if lam else None, fa.alpha if lam else None)
        assert torch.equal(fb.radii, fa.radii)
        for gr, gq in zip(ob.param_groups, oa.param_groups):
            for p, q in zip(gr["params"], gq["params"]):
                for k in ("exp_avg", "exp_avg_sq"):
                    a, b = ob.state[p][k], oa.state[q][k]
                    scale = float(b.abs().max()) + 1e-30
                    assert float((a - b).abs().max()) <= 1e-3 * scale + 1e-12, f"{gr.get('name')} {k}"
    assert fa.captures == 1 and fb.captures == 1


def test_prefetching_pair_with_store_host_inputs():
    """Two frames with host_inputs prefetch each other's staged camera and frame ids inside their graphs; each
    replay decodes the frame that was staged for it, and its loss is the eager one."""
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    from gaussianavatars_b200.renderer import render
    g = _g()
    sc, _ = RM._single_view_setup()
    pc = TG._model(sc)
    cams = [sc["cam"], syn.orbit_camera(sc["W"], sc["H"], r=1.1, fovy_deg=22.0, azimuth_deg=-20.0)]
    store = g.FrameStore(sc["W"], sc["H"], sc["bg"], DEV)
    rgbas = RM._rgba(5, sc["H"], sc["W"], seed=60)
    store.add_rgba(rgbas)
    frames = []
    for k in range(2):
        f = GraphedFrame(pc, sc["W"], sc["H"], sc["cam"].FoVx, sc["cam"].FoVy, sc["bg"], loss="l1_u8",
                         host_inputs=True, frames=store, lambda_mask=LAM, per_camera_fov=True, warm_cameras=cams)
        assert f.frames_stage.shape == (1,) and f.frames_stage.is_pinned() and f.gt_stage is None
        f.set_inputs(verts=sc["verts"].to(DEV))
        frames.append(f)
    frames[0].prefetch_for(frames[1])
    frames[1].prefetch_for(frames[0])
    for f in frames:
        f.capture()
    order = [3, 1, 4, 0, 2]
    frames[0].cam_stage.copy_(camera_block(cams[0], fov=True))
    frames[0].stage_frames(order[0])
    frames[0].upload_staged()
    bg = sc["bg"].to(DEV)
    for i in range(5):
        cur, nxt = frames[i % 2], frames[(i + 1) % 2]
        torch.cuda.synchronize()
        if i + 1 < 5:
            nxt.cam_stage.copy_(camera_block(cams[(i + 1) % 2], fov=True))
            nxt.stage_frames(order[i + 1])
        cur.run(check=True)
        torch.cuda.synchronize()
        gt, mask = g.composite_rgba(rgbas[order[i]].to(DEV), bg)
        assert torch.equal(cur.gt, gt) and torch.equal(cur.mask, mask), f"step {i}: decoded frame differs"
        pc.update_mesh_properties(sc["verts"].to(DEV))
        out = render(cams[i % 2].to(DEV), pc, TG.Pipe, bg, depth_alpha=True)
        ref = float(g.l1_loss_u8(out["render"], gt)) + float(g.l1_loss_u8(out["alpha"], mask)) * LAM
        assert torch.equal(cur.image, out["render"].detach()), f"step {i}"
        assert abs(float(cur.loss_host) - ref) <= 1e-6 * ref
    assert all(f.captures == 1 for f in frames)
    # set_inputs on a host-input frame uploads the ids on the copy stream
    frames[0].set_inputs(frames=2)
    frames[0].run(check=True)
    torch.cuda.synchronize()
    assert torch.equal(frames[0].gt, g.composite_rgba(rgbas[2].to(DEV), bg)[0])


def test_overflowing_store_replay_applies_no_step_and_check_recovers():
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.graph import camera_block
    g = _g()
    sc, _ = RM._single_view_setup()
    pc = TG._trainable(sc)
    other = syn.orbit_camera(sc["W"], sc["H"], r=1.0, fovy_deg=20.0, azimuth_deg=25.0)
    store = g.FrameStore(sc["W"], sc["H"], sc["bg"], DEV)
    rgba = RM._rgba(2, sc["H"], sc["W"], seed=70)
    store.add_rgba(rgba)
    fr = RM._single_frame(pc, sc, frames=store, lambda_mask=LAM,
                          warm_cameras=[camera_block(sc["cam"]), camera_block(other)])
    fr.set_inputs(frames=1)
    pc.optimizer.init_state()
    snap = TG._snapshot(pc)
    fr.capture(capacity=4096)
    fr.run(check=False)
    assert fr.overflowed(wait=True), "an overflowing replay was not flagged"
    TG._assert_state_equal(pc, snap, "overflowing replay")
    img, alpha, loss, pc_e = RM._eager_mask_iteration_single(sc, snap, sc["verts"], rgba[1].to(DEV),
                                                             pc.active_sh_degree)
    fr.run(check=True)
    torch.cuda.synchronize()
    assert fr.captures == 2 and not fr.overflowed(wait=True)
    assert torch.equal(fr.image, img) and torch.equal(fr.alpha, alpha)
    assert abs(float(fr.loss) - loss) <= 1e-6 * loss
    TG._grads_close([p.grad for p in pc.parameters()], [p.grad for p in pc_e.parameters()])
    RM._check_step_exact(fr, pc, snap, "regrown replay")


def test_one_recapture_after_the_store_grows_and_none_for_new_ids():
    g = _g()
    sc, _ = RM._single_view_setup()
    pc = TG._trainable(sc)
    store = g.FrameStore(sc["W"], sc["H"], sc["bg"], DEV)
    rgba = RM._rgba(8, sc["H"], sc["W"], seed=80)
    store.add_rgba(rgba[:2])
    fr = RM._single_frame(pc, sc, frames=store)
    bg = sc["bg"].to(DEV)
    want = g.composite_rgba(rgba.to(DEV), bg)
    for i in (0, 1, 0, 1):
        fr.set_inputs(frames=i)
        fr.run(check=True)
        torch.cuda.synchronize()
        assert torch.equal(fr.gt, want[0][i]) and torch.equal(fr.mask, want[1][i])
    assert fr.captures == 1
    ptrs = store.pointers()
    store.add_rgba(rgba[2:5])          # the arena grows: one re-capture
    assert store.pointers() != ptrs
    for i in (4, 2, 3):
        fr.set_inputs(frames=i)
        fr.run(check=True)
        torch.cuda.synchronize()
        assert torch.equal(fr.gt, want[0][i]) and torch.equal(fr.mask, want[1][i])
    assert fr.captures == 2
