"""-m gpu: the device-resident view schedule (csrc/schedule.cu, schedule.ViewSchedule, GraphedFrame(schedule=),
GraphedEval(schedule=, frames=)).

The L1 loss, the blend backward and the face-frame backward sum with float atomics, so two runs agree bit for bit
only in what is deterministic; every quantity is held to the strictest standard it admits:
  * a frozen model (optimizer=None, densify_stats=True), K = 1 and 4, FLAME head, frames=store, a rig of mixed FoVs:
    after every run_iterations(1) the camera table, timestep, frame ids, decoded gt / mask, image and radii equal the
    host-driven replay of order[i]; one run_iterations(n) across an epoch boundary gives denom and max_radii2D
    exactly, xyz_gradient_accum and the loss log within a stated tolerance, over records whose losses differ by far
    more than it;
  * training (capturable Adam with lr_schedule, statistics, regularisers, lambda_mask), K = 1 and 16: the state after
    n scheduled iterations against n host-driven ones, to the standard of tests/test_gpu_multiview_train.py; every
    Adam step counter and the cursor equal n;
  * an overflow mid-run: one re-capture, the cursor, step counters and denom of the run without overflow, every log
    row written once;
  * a re-capture between runs (densify_and_prune, oneupSHdegree): the cursor and the log persist;
  * GraphedEval(schedule=, frames=): rows equal the host-fed rows bit for bit, K = 1 and 4, source float and u8, and
    an overflowed record redone by run_all;
  * the device guard: a sampler launched with cursor = L writes nothing and raises `exhausted`; the commit then
    leaves the cursor alone."""
import ctypes as C

import pytest
import torch

from tests import test_gpu_multiview_train as MV
from tests.test_gpu_camera_fov import _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
H_S, W_S = 550, 802
T_MODEL = 6   # timesteps of MV._flame_trainable's head
LOSS_RTOL = 1e-4


def _g():
    import gaussianavatars_b200 as g
    return g


def _level_frames(R, K, H, W, seed):
    """(R*K, H, W, 4) opaque RGBA frames, record r at its own grey level (plus noise): the records' losses differ by
    far more than LOSS_RTOL."""
    gen = torch.Generator().manual_seed(seed)
    rgba = torch.randint(0, 24, (R * K, H, W, 4), generator=gen, dtype=torch.uint8)
    for r in range(R):
        rgba[r * K:(r + 1) * K, ..., :3] += 12 + int(200 * r / max(R - 1, 1))
    rgba[..., 3] = 255
    return rgba


def _records(R, K, seed=0):
    """R records of K rig cameras (mixed FoVs), timestep r % T, frame ids r*K .. r*K+K-1, and a store holding them."""
    rig = _rig(W_S, H_S, n=max(K + R - 1, 2))
    groups = [rig[r:r + K] for r in range(R)]
    ts = [(3 * r + 1) % T_MODEL for r in range(R)]
    ids = [[r * K + k for k in range(K)] for r in range(R)]
    store = _g().FrameStore(W_S, H_S, torch.ones(3), DEV)
    store.add_rgba(_level_frames(R, K, H_S, W_S, seed))
    return groups, ts, ids, store


def _schedule(groups, ts, ids, K, order):
    cams = [g[0] for g in groups] if K == 1 else groups
    flat = [i[0] for i in ids] if K == 1 else ids
    return _g().ViewSchedule(cams, timesteps=ts, frames=flat, order=order, device=DEV)


def _host_inputs(fr, groups, ts, ids, r):
    pose = dict(cameras=groups[r]) if fr.K > 1 else dict(camera=groups[r][0])
    fr.set_inputs(timestep=ts[r], frames=ids[r] if fr.K > 1 else ids[r][0], **pose)


def _zero_stats(pc):
    for n in ("xyz_gradient_accum", "denom", "max_radii2D"):
        getattr(pc, n).zero_()


# ---- a frozen model: everything deterministic is bit for bit ------------------------------------------------------
@pytest.mark.parametrize("K", [1, 4])
def test_frozen_scheduled_replays_equal_the_host_driven_replays(K):
    from gaussianavatars_b200.graph import GraphedFrame
    g = _g()
    pc, _ = MV._flame_trainable()
    R, n = 5, 8   # an epoch of 5 and 3 records of the next
    groups, ts, ids, store = _records(R, K)
    order = g.epoch_order(R, n, torch.Generator().manual_seed(7))
    s = _schedule(groups, ts, ids, K, order)
    warm = groups[:2] if K > 1 else [c[0] for c in groups[:2]]
    common = dict(loss="l1_u8", densify_stats=True, views_per_replay=K, frames=store, warm_cameras=warm,
                  per_camera_fov=True)
    fa = GraphedFrame(pc, W_S, H_S, 1.0, 1.0, torch.ones(3), schedule=s, **common)
    fb = GraphedFrame(pc, W_S, H_S, 1.0, 1.0, torch.ones(3), **common)
    for i in range(n):
        assert fa.run_iterations(1) == 1
        r = s.record(i)
        _host_inputs(fb, groups, ts, ids, r)
        fb.run(check=True)
        torch.cuda.synchronize()
        what = f"K={K} iteration {i} record {r}"
        assert int(fa.cursor) == i + 1, what
        assert torch.equal(fa.cam, fb.cam), f"{what}: camera table"
        assert torch.equal(fa.timestep, fb.timestep) and int(fa.timestep) == ts[r], f"{what}: timestep"
        assert torch.equal(fa.frame_ids, fb.frame_ids) and fa.frame_ids.tolist() == ids[r], f"{what}: frame ids"
        assert torch.equal(fa.gt, fb.gt) and torch.equal(fa.mask, fb.mask), f"{what}: decoded frames"
        assert torch.equal(fa.image, fb.image) and torch.equal(fa.radii, fb.radii), f"{what}: image / radii"
    # one run across the epoch boundary against n host-driven replays
    fa.set_cursor(0)
    _zero_stats(pc)
    assert fa.run_iterations(n) == n and int(fa.cursor) == n
    got = {k: getattr(pc, k).clone() for k in ("xyz_gradient_accum", "denom", "max_radii2D")}
    log = fa.loss_history()
    _zero_stats(pc)
    ref = []
    for i in range(n):
        _host_inputs(fb, groups, ts, ids, s.record(i))
        fb.run(check=True)
        ref.append(float(fb.loss))
    ref = torch.tensor(ref)
    assert torch.equal(got["denom"], pc.denom) and torch.equal(got["max_radii2D"], pc.max_radii2D)
    a, b = got["xyz_gradient_accum"], pc.xyz_gradient_accum
    assert float((a - b).abs().max()) <= 1e-4 * float(b.abs().max()), "xyz_gradient_accum"
    rel = ((log - ref).abs() / ref.abs()).max()
    per_record = sorted({s.record(i): float(ref[i]) for i in range(n)}.values())
    gap = min(abs(x - y) / max(x, y) for x, y in zip(per_record, per_record[1:]))
    print(f"[schedule] K={K}: loss log vs host {float(rel):.1e} (tolerance {LOSS_RTOL:.0e}); records apart >= {gap:.2e}")
    assert len(per_record) == R and gap >= 100 * LOSS_RTOL, "the records' losses must tell them apart"
    assert float(rel) <= LOSS_RTOL
    assert fa.captures == 1 and fb.captures == 1


# ---- training ------------------------------------------------------------------------------------------------------
def _scheduled_trainable():
    """MV._flame_trainable with an lr_schedule on the position group."""
    g = _g()
    pc, opt = MV._flame_trainable()
    opt.param_groups[0]["lr_schedule"] = g.expon_lr_schedule(lr_init=1.6e-4, lr_final=1.6e-6, lr_delay_mult=0.01,
                                                             max_steps=30)
    return pc, opt


def _train_frame(pc, opt, K, store, **kw):
    from gaussianavatars_b200.graph import GraphedFrame
    return GraphedFrame(pc, W_S, H_S, 1.0, 1.0, torch.ones(3), loss="photometric", regularizers={}, optimizer=opt,
                        densify_stats=True, views_per_replay=K, frames=store, lambda_mask=0.1, per_camera_fov=True,
                        **kw)


def _compare_training(pa, oa, pb, ob, n, what):
    for gr, gq in zip(oa.param_groups, ob.param_groups):
        for p, q in zip(gr["params"], gq["params"]):
            assert float(oa.state[p]["step"]) == n and torch.equal(oa.state[p]["step"], ob.state[q]["step"]), what
            d = (p.detach() - q.detach()).abs()
            bound = 2 * n * max(gr["lr"], 1.6e-4 if gr.get("lr_schedule") else 0.0)
            frac = float((d > 0.25 * bound + 1e-7).float().mean())
            assert frac <= 1e-2, f"{what}: {gr.get('name')} {frac:.1e}"
    for k in ("denom", "max_radii2D"):
        assert float((getattr(pa, k) != getattr(pb, k)).float().mean()) <= 1e-3, f"{what}: {k}"
    a, b = pa.xyz_gradient_accum, pb.xyz_gradient_accum
    assert float(((a - b).abs() > 1e-3 * b.abs() + 1e-6 * float(b.abs().max())).float().mean()) <= 1e-2, what


@pytest.mark.parametrize("K", [1, 16])
def test_scheduled_training_equals_host_driven_training(K):
    g = _g()
    R, n = (4, 6) if K == 1 else (3, 4)
    groups, ts, ids, store = _records(R, K, seed=K)
    order = g.epoch_order(R, n, torch.Generator().manual_seed(K))
    s = _schedule(groups, ts, ids, K, order)
    (pa, oa), (pb, ob) = _scheduled_trainable(), _scheduled_trainable()
    fa = _train_frame(pa, oa, K, store, schedule=s)
    warm = [groups[r] if K > 1 else groups[r][0] for r in s.warm_records()]
    fb = _train_frame(pb, ob, K, store, warm_cameras=warm)
    assert fa.run_iterations(n) == n
    ref = []
    for i in range(n):
        _host_inputs(fb, groups, ts, ids, s.record(i))
        fb.run(check=True)
        ref.append(float(fb.loss))
    torch.cuda.synchronize()
    assert int(fa.cursor) == n and fa.captures == 1 and fb.captures == 1
    _compare_training(pa, oa, pb, ob, n, f"K={K}")
    log, ref = fa.loss_history(), torch.tensor(ref)
    print(f"[schedule] training K={K}: loss log vs host max rel {float(((log - ref).abs() / ref).max()):.1e}")
    assert float(((log - ref).abs() / ref).max()) <= 1e-3


def test_overflow_mid_run_recaptures_once_and_resumes_at_the_record():
    """A capacity that fits the first iterations of the order but not a later one: run_iterations(n) overflows
    mid-run, regrows once and replays from that iteration; the cursor and every step counter equal the run that never
    overflowed, denom is that run's, and every log row is written exactly once (the records' losses tell them
    apart)."""
    K, R, n = 1, 4, 6
    groups, ts, ids, store = _records(R, K, seed=3)
    s = _schedule(groups, ts, ids, K, [3, 2, 1, 0, 1, 3])   # the widest FoV first: fewer instances
    (pa, oa), (pb, ob) = _scheduled_trainable(), _scheduled_trainable()
    fb = _train_frame(pb, ob, K, store, schedule=s)
    counts = []
    for i in range(n):   # the run without overflow, and what each iteration needs
        assert fb.run_iterations(1) == 1
        counts.append(fb.counters()["num_rendered"])
    assert fb.captures == 1
    j = next((i for i in range(1, n) if counts[i] > max(counts[:i]) * 1.02), None)
    assert j is not None, f"no iteration needs more instances than the ones before it: {counts}"
    cap = (max(counts[:j]) + counts[j]) // 2
    fa = _train_frame(pa, oa, K, store, schedule=s)
    fa.capture(capacity=cap)
    assert fa.run_iterations(n) == n
    torch.cuda.synchronize()
    print(f"[schedule] overflow: instances per iteration {counts}, capacity {cap}, first overflow at iteration {j}")
    assert fa.captures == 2, "the run must re-capture exactly once"
    assert int(fa.cursor) == n and not fa.overflowed()
    for gr, gq in zip(oa.param_groups, ob.param_groups):
        for p, q in zip(gr["params"], gq["params"]):
            assert float(oa.state[p]["step"]) == n and torch.equal(oa.state[p]["step"], ob.state[q]["step"])
    assert float((pa.denom != pb.denom).float().mean()) <= 1e-3, "denom"
    assert int(pa.denom.max()) == int(pb.denom.max()) <= n
    log, ref = fa.loss_history(), fb.loss_history()
    assert not torch.isnan(log).any(), "a log row was skipped"
    assert float(((log - ref).abs() / ref).max()) <= 1e-3, "a log row holds another iteration's loss"


def test_recapture_between_runs_keeps_the_cursor_and_the_log():
    """oneupSHdegree and densify_and_prune between runs re-capture; the cursor and the log are the frame's and the
    next run continues the order."""
    g = _g()
    K, R = 1, 4
    groups, ts, ids, store = _records(R, K, seed=5)
    s = _schedule(groups, ts, ids, K, g.epoch_order(R, 9, torch.Generator().manual_seed(2)))
    pc, opt = _scheduled_trainable()
    pc.optimizer = opt   # what densify_and_prune reads beyond the model: train.py's GaussianModel attributes
    pc.percent_dense = 0.01
    pc.binding_counter = torch.bincount(pc.binding.long(), minlength=pc.faces.shape[0]).to(torch.int32)
    pc.active_sh_degree = 0
    fr = _train_frame(pc, opt, K, store, schedule=s)
    assert fr.run_iterations(3) == 3
    log3 = fr.loss_history(0, 3)
    cursor_addr, log_addr = fr.cursor.data_ptr(), fr.losses.data_ptr()
    pc.active_sh_degree += 1   # oneupSHdegree
    assert fr.run_iterations(3) == 3 and fr.captures == 2 and int(fr.cursor) == 6
    P0 = pc._xyz.shape[0]
    grads = pc.xyz_gradient_accum / pc.denom
    thr = float(torch.nan_to_num(grads, 0.0).quantile(0.9))
    info = g.densify_and_prune(pc, thr, 0.005, 1.0, None, generator=torch.Generator(DEV).manual_seed(3))
    assert info["P_out"] != P0
    assert fr.run_iterations(3) == 3 and fr.captures == 3 and int(fr.cursor) == 9
    assert fr.cursor.data_ptr() == cursor_addr and fr.losses.data_ptr() == log_addr
    log = fr.loss_history()
    assert torch.equal(log[:3], log3) and not torch.isnan(log).any()
    assert float(opt.state[pc._xyz]["step"]) == 9
    with pytest.raises(ValueError, match="could run past"):
        fr.run_iterations(1)


# ---- evaluation ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("source", ["float", "u8"])
@pytest.mark.parametrize("K", [1, 4])
def test_scheduled_eval_rows_equal_the_host_fed_rows(K, source):
    from gaussianavatars_b200.graph import GraphedEval
    R = 4
    groups, ts, ids, store = _records(R, K, seed=20 + K)
    s = _schedule(groups, ts, ids, K, None)
    pc, _ = MV._flame_trainable()
    warm = groups[:2] if K > 1 else [c[0] for c in groups[:2]]
    common = dict(views=R * K, source=source, views_per_replay=K, warm_cameras=warm)
    ea = GraphedEval(pc, W_S, H_S, torch.ones(3), schedule=s, frames=store, **common)
    eb = GraphedEval(pc, W_S, H_S, torch.ones(3), **common)
    assert ea.run_all() == R and int(ea.cursor) == R
    for r in range(R):
        gt, _ = store.decode(ids[r])
        pose = dict(cameras=groups[r]) if K > 1 else dict(camera=groups[r][0])
        eb.set_inputs(timestep=ts[r], gt_u8=gt if K > 1 else gt[0], view=r * K, **pose)
        eb.run(check=True)
    a, b = ea.scores(), eb.scores()
    assert torch.equal(a["per_view"], b["per_view"]), "scheduled rows differ from the host-fed rows"
    # reset rewinds; a second pass writes the same rows
    ea.reset()
    assert int(ea.cursor) == 0 and ea.run_all() == R
    assert torch.equal(ea.scores()["per_view"], b["per_view"])


def test_scheduled_eval_redoes_an_overflowed_record():
    from gaussianavatars_b200.graph import GraphedEval
    K, R = 1, 4
    groups, ts, ids, store = _records(R, K, seed=30)
    s = _schedule(groups, ts, ids, K, None)
    pc, _ = MV._flame_trainable()
    ref = GraphedEval(pc, W_S, H_S, torch.ones(3), views=R, schedule=s, frames=store)
    ref.run_all()
    want = ref.scores()["per_view"]
    ev = GraphedEval(pc, W_S, H_S, torch.ones(3), views=R, schedule=s, frames=store)
    ev.capture(capacity=4096)
    assert ev.run_all(check=False) is None
    torch.cuda.synchronize()
    assert ev.overflowed() and int(ev.cursor) == 0, "the first record must overflow a 4096-instance capacity"
    assert torch.isnan(ev.table).all(), "an overflowed replay wrote a row"
    with pytest.raises(ValueError, match="could run past"):
        ev.run()   # the host bound: every record was enqueued already
    ev.set_cursor(0)   # the cursor the device holds: the overflowed record
    assert ev.run_all() == R and ev.captures == 2
    assert torch.equal(ev.scores()["per_view"], want)


# ---- the device guard ----------------------------------------------------------------------------------------------
def test_sampler_past_the_order_writes_nothing_and_the_commit_holds():
    from gaussianavatars_b200 import _native as N
    R, K, L = 3, 2, 5
    cams = torch.randn(R, K, 37, device=DEV)
    ts = torch.tensor([2, 0, 1], dtype=torch.int32, device=DEV)
    fids = torch.arange(R * K, dtype=torch.int32, device=DEV).reshape(R, K)
    order = torch.tensor([2, 1, 0, 0, 1], dtype=torch.int32, device=DEV)
    cursor = torch.tensor([L], dtype=torch.int32, device=DEV)
    cam_out = torch.full((K, 37), 7.0, device=DEV)
    t_out = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    ids_out = torch.full((K,), -7, dtype=torch.int32, device=DEV)
    rows_out = torch.full((K,), -7, dtype=torch.int32, device=DEV)
    exhausted = torch.zeros(1, dtype=torch.int32, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    loss = torch.full((), 3.5, device=DEV)
    losses = torch.full((L,), float("nan"), device=DEV)
    L_ = N.lib()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def sample():
        N.check(L_.gab200_schedule_sample(R, K, L, cams.data_ptr(), ts.data_ptr(), fids.data_ptr(), order.data_ptr(),
                                          cursor.data_ptr(), cam_out.data_ptr(), t_out.data_ptr(), ids_out.data_ptr(),
                                          rows_out.data_ptr(), exhausted.data_ptr(), stream), "sample")

    def commit():
        N.check(L_.gab200_schedule_commit(L, flag.data_ptr(), exhausted.data_ptr(), loss.data_ptr(),
                                          losses.data_ptr(), cursor.data_ptr(), stream), "commit")

    sample()
    commit()
    torch.cuda.synchronize()
    assert int(exhausted) == 1 and int(cursor) == L
    assert bool((cam_out == 7.0).all()) and int(t_out) == -7 and ids_out.tolist() == [-7, -7]
    assert rows_out.tolist() == [-7, -7] and torch.isnan(losses).all()
    # in range: record order[c] lands, the commit logs and advances; an overflow flag holds the cursor
    cursor.fill_(1)
    exhausted.zero_()
    sample()
    commit()
    torch.cuda.synchronize()
    assert torch.equal(cam_out, cams[1]) and int(t_out) == 0 and ids_out.tolist() == [2, 3]
    assert rows_out.tolist() == [2, 3] and int(cursor) == 2 and float(losses[1]) == 3.5 and int(exhausted) == 0
    flag.fill_(1)
    sample()
    commit()
    torch.cuda.synchronize()
    assert torch.equal(cam_out, cams[0]) and int(cursor) == 2 and torch.isnan(losses[2])
