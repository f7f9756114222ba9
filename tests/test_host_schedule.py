"""CPU: the device-resident view schedule's surface (schedule.ViewSchedule, epoch_order, gab200_schedule_sample /
gab200_schedule_commit, GraphedFrame(schedule=), GraphedEval(schedule=, frames=)) -- construction and every refusal,
the per-epoch permutation semantics, the exports and header declarations, the C ABI's argument refusals, and the
host bound of a scheduled run.  No device: the schedule's tensors stay on the CPU and the frames stub their capture
as tests/test_host_frame_store.py does."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

from tests.test_host_frame_store import _store, no_device  # noqa: F401  (no_device: a fixture)

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PARAMS = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
W, H = 40, 24
SIGNATURES = {
    "gab200_schedule_sample": ["records", "views", "length", "cams", "timesteps", "frame_ids", "order", "cursor",
                               "cam_out", "timestep_out", "ids_out", "rows_out", "exhausted", "stream"],
    "gab200_schedule_commit": ["length", "overflow_flag", "exhausted", "loss", "losses", "cursor", "stream"],
}


@pytest.fixture()
def cpu_schedule(monkeypatch):
    """Schedules whose tensors stay on the CPU (the library has no CPU path; the checks are host code)."""
    from gaussianavatars_b200 import schedule as S
    monkeypatch.setattr(S, "_cuda_device", lambda device=None: torch.device("cpu"))
    return S


def _cams(n, w=W, h=H):
    from gaussianavatars_b200 import synthetic as syn
    return [syn.orbit_camera(w, h, r=1.0 + 0.01 * i, fovy_deg=18.0 + i, azimuth_deg=5.0 * i) for i in range(n)]


# ---- exports and the C ABI -----------------------------------------------------------------------------------------
def test_exported_and_declared():
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    for name, params in SIGNATURES.items():
        assert name in N.EXPORTED_SYMBOLS and hasattr(L, name)
        decl = re.search(r"int32_t " + name + r"\(([^)]*)\);", hdr)
        assert decl is not None, name
        assert [p.split()[-1].lstrip("*") for p in decl.group(1).split(",")] == params, name
        assert len(getattr(L, name).argtypes) == len(params)
        ints = [p for p in re.split(r",\s*", decl.group(1)) if p.startswith("int32_t ")]
        assert getattr(L, name).argtypes[:len(ints)] == [C.c_int32] * len(ints), name
        assert all(t is C.c_void_p for t in getattr(L, name).argtypes[len(ints):]), name
    for n in ("ViewSchedule", "epoch_order"):
        assert n in g.__all__ and getattr(g, n).__module__ == "gaussianavatars_b200.schedule"
    assert L.gab200_abi_version() == 3


def test_c_abi_refusals_before_any_device_work():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    buf = (C.c_uint8 * 256)()
    p = C.cast(buf, C.c_void_p)
    invalid = -1
    ok = [p] * 10   # cams, timesteps, frame_ids, order, cursor, cam_out, timestep_out, ids_out, rows_out, exhausted
    for dims in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (-1, 1, 1), (1, 65536, 1), (2 ** 16, 2 ** 15, 1)):
        assert L.gab200_schedule_sample(*dims, *ok, None) == invalid, dims
    for k in (0, 3, 4, 5, 9):   # cams, order, cursor, cam_out or exhausted missing
        args = list(ok)
        args[k] = None
        assert L.gab200_schedule_sample(1, 1, 1, *args, None) == invalid, k
    for table, out in ((1, 6), (2, 7)):   # an output without the table it copies
        args = list(ok)
        args[table] = None
        assert L.gab200_schedule_sample(1, 1, 1, *args, None) == invalid
    # commit: length, overflow_flag, exhausted, loss, losses, cursor
    assert L.gab200_schedule_commit(0, p, p, p, p, p, None) == invalid
    assert L.gab200_schedule_commit(1, p, None, p, p, p, None) == invalid
    assert L.gab200_schedule_commit(1, p, p, p, p, None, None) == invalid
    assert L.gab200_schedule_commit(1, p, p, None, p, p, None) == invalid   # a log without a loss


# ---- epoch_order ---------------------------------------------------------------------------------------------------
def test_epoch_order_is_one_permutation_per_epoch_truncated():
    from gaussianavatars_b200.schedule import epoch_order
    R, n = 7, 7 * 3 + 4
    o = epoch_order(R, n, torch.Generator().manual_seed(3))
    assert o.dtype == torch.int32 and o.shape == (n,)
    epochs = [o[i:i + R].tolist() for i in range(0, n, R)]
    for e in epochs[:3]:
        assert sorted(e) == list(range(R))
    assert len(epochs[3]) == 4 and len(set(epochs[3])) == 4   # the truncated last epoch: a prefix of a permutation
    assert len({tuple(e) for e in epochs[:3]}) == 3            # every epoch its own order
    assert torch.equal(o, epoch_order(R, n, torch.Generator().manual_seed(3)))
    assert not torch.equal(o, epoch_order(R, n, torch.Generator().manual_seed(4)))
    # the same permutations torch.randperm draws from the generator, epoch after epoch
    g = torch.Generator().manual_seed(3)
    want = torch.cat([torch.randperm(R, generator=g) for _ in range(4)])[:n]
    assert torch.equal(o, want.to(torch.int32))
    assert epoch_order(R, 0).numel() == 0 and epoch_order(1, 3).tolist() == [0, 0, 0]
    for bad in ((0, 3), (3, -1)):
        with pytest.raises(ValueError, match="epoch_order needs"):
            epoch_order(*bad)


# ---- ViewSchedule --------------------------------------------------------------------------------------------------
def test_schedule_construction(cpu_schedule):
    from gaussianavatars_b200.graph import camera_block
    from gaussianavatars_b200.renderer import camera_table
    S = cpu_schedule
    cams = _cams(5)
    s = S.ViewSchedule(cams, timesteps=[0, 4, 2, 1, 3], frames=[4, 3, 2, 1, 0], order=[1, 1, 0, 4])
    assert (s.R, s.K, s.L, s.W, s.H) == (5, 1, 4, W, H) and len(s) == 4
    assert s.cams.shape == (5, 1, 37) and s.cams.dtype == torch.float32
    assert torch.equal(s.cams[2, 0], camera_block(cams[2], fov=True))
    assert s.timesteps.dtype == torch.int32 and s.timesteps.tolist() == [0, 4, 2, 1, 3]
    assert s.frame_ids.shape == (5, 1) and s.frame_ids[:, 0].tolist() == [4, 3, 2, 1, 0]
    assert s.order.dtype == torch.int32 and s.order.tolist() == [1, 1, 0, 4] and s.record(3) == 4
    assert s.max_timestep == 4 and s.max_frame_id == 4
    # groups of K cameras: the rows of camera_table; the identity order by default
    groups = [cams[0:2], cams[2:4], cams[3:5]]
    g = S.ViewSchedule(groups, frames=[[0, 1], [2, 3], [3, 4]])
    assert (g.R, g.K, g.L) == (3, 2, 3) and g.order.tolist() == [0, 1, 2]
    assert torch.equal(g.cams[1], camera_table(groups[1], "cpu")) and g.frame_ids.tolist() == [[0, 1], [2, 3], [3, 4]]
    # a tensor: (R, 37) or (R, K, 37); no image size
    t = S.ViewSchedule(g.cams.clone())
    assert (t.R, t.K, t.W, t.H) == (3, 2, None, None)
    assert S.ViewSchedule(s.cams[:, 0].clone()).K == 1
    # the warm-up records: up to 16 spread over the table
    assert S.ViewSchedule(_cams(1)).warm_records() == [0]
    big = S.ViewSchedule(torch.zeros(40, 37))
    w = big.warm_records()
    assert len(w) == 16 and w[0] == 0 and w[-1] == 39 and w == sorted(set(w))
    assert S.ViewSchedule(torch.zeros(5, 37)).warm_records() == [0, 1, 2, 3, 4]


def test_schedule_refusals(cpu_schedule):
    S = cpu_schedule
    cams = _cams(3)
    with pytest.raises(ValueError, match="at least one record"):
        S.ViewSchedule([])
    with pytest.raises(ValueError, match="one image size"):
        S.ViewSchedule(cams[:2] + _cams(1, w=W + 2))
    with pytest.raises(ValueError, match="the same number of cameras"):
        S.ViewSchedule([cams[:2], cams[:1]])
    with pytest.raises(ValueError, match=r"\(R, K, 37\)"):
        S.ViewSchedule(torch.zeros(3, 2, 35))
    with pytest.raises(ValueError, match="must be finite"):
        S.ViewSchedule(torch.full((2, 37), float("nan")))
    with pytest.raises(ValueError, match="order entries index the schedule's 3 records"):
        S.ViewSchedule(cams, order=[0, 3])
    with pytest.raises(ValueError, match="order entries index"):
        S.ViewSchedule(cams, order=[-1])
    for bad in ([], [0.0, 1.0], [[0, 1]], [True]):
        with pytest.raises(ValueError, match="order must be"):
            S.ViewSchedule(cams, order=bad)
    with pytest.raises(ValueError, match="timesteps must hold 3 values"):
        S.ViewSchedule(cams, timesteps=[0, 1])
    with pytest.raises(ValueError, match="timesteps must be non-negative"):
        S.ViewSchedule(cams, timesteps=[0, -1, 2])
    with pytest.raises(ValueError, match="timesteps must hold integers"):
        S.ViewSchedule(cams, timesteps=[0.0, 1.0, 2.0])
    with pytest.raises(ValueError, match="frames must hold 3x2 values"):
        S.ViewSchedule([cams[:2]] * 3, frames=[0, 1, 2])


def test_a_schedule_lives_on_a_cuda_device():
    from gaussianavatars_b200 import schedule as S
    with pytest.raises(RuntimeError, match="no CPU path"):
        S.ViewSchedule(torch.zeros(2, 37), device="cpu")


# ---- frames built on a schedule ------------------------------------------------------------------------------------
def _model(P=4, verts=False, T=None):
    pc = SimpleNamespace(active_sh_degree=0, binding=None, verts_rest=torch.zeros(5, 3) if verts else None)
    for n in PARAMS:
        setattr(pc, n, torch.nn.Parameter(torch.zeros(P, 3)))
    pc.parameters = lambda: [getattr(pc, n) for n in PARAMS]
    if T is not None:   # a FLAME head of T timesteps (only its shape is read on the host)
        pc.flame = object()
        pc.flame_param = {"expr": torch.zeros(T, 10)}
    return pc


def _frame(s, store=None, K=1, pc=None, **kw):
    from gaussianavatars_b200.graph import GraphedFrame
    fr = GraphedFrame(pc if pc is not None else _model(), W, H, 0.7, 0.5, torch.zeros(3), frames=store,
                      views_per_replay=K, schedule=s, **kw)
    fr._learn_capacity = lambda: (0, (0, 0))
    fr._body = lambda *a, **k: None
    return fr


def test_graphed_frame_schedule_refusals(cpu_schedule, no_device):
    S = cpu_schedule
    cams = _cams(3)
    store = _store(n=3)
    s = S.ViewSchedule(cams, frames=[0, 1, 2])
    fr = _frame(s, store)
    assert fr.per_camera_fov and fr.cam.shape == (37,) and fr.cursor.tolist() == [0] and fr.exhausted.tolist() == [0]
    assert fr.losses.shape == (3,) and torch.isnan(fr.losses).all()
    assert [b for b, _ in fr._warm_pairs] and all(t is None for _, t in fr._warm_pairs)
    for kw, msg in ((dict(host_inputs=True), "host_inputs=True stages them"),
                    (dict(rgba=True), "nothing on the device holds the RGBA frames"),
                    (dict(loss="dL_dimage"), "loss='dL_dimage'")):
        with pytest.raises(ValueError, match=msg):
            _frame(s, store, **kw)
    with pytest.raises(ValueError, match="nothing on the device holds the RGBA frames"):
        _frame(S.ViewSchedule(cams), None, rgba=True)
    with pytest.raises(ValueError, match="posed by host vertices"):
        _frame(S.ViewSchedule(cams, frames=[0, 1, 2]), store, pc=_model(verts=True))
    with pytest.raises(ValueError, match="must be a gaussianavatars_b200.ViewSchedule"):
        _frame(object(), store)
    with pytest.raises(ValueError, match="the schedule's records hold 1 cameras, this GraphedFrame renders 2"):
        _frame(s, store, K=2)
    with pytest.raises(ValueError, match="the schedule's cameras are 42x24"):
        _frame(S.ViewSchedule(_cams(2, w=W + 2), frames=[0, 1]), store)
    with pytest.raises(ValueError, match="needs a schedule with frames="):
        _frame(S.ViewSchedule(cams), store)
    with pytest.raises(ValueError, match="reads no frame store"):
        _frame(s, None)
    with pytest.raises(ValueError, match="frame ids reach 3, the store holds 3"):
        _frame(S.ViewSchedule(cams, frames=[0, 3, 1]), store)
    with pytest.raises(ValueError, match="no FLAME head"):
        _frame(S.ViewSchedule(cams, timesteps=[0, 0, 0], frames=[0, 1, 2]), store)
    with pytest.raises(ValueError, match="needs timesteps="):
        _frame(s, store, pc=_model(T=4))
    with pytest.raises(ValueError, match="timesteps reach 4, the model has 4"):
        _frame(S.ViewSchedule(cams, timesteps=[0, 4, 1], frames=[0, 1, 2]), store, pc=_model(T=4))
    flame = _frame(S.ViewSchedule(cams, timesteps=[3, 0, 2], frames=[0, 1, 2]), store, pc=_model(T=4))
    assert flame.timestep is not None and [t for _, t in flame._warm_pairs] == [3, 0, 2]
    warm = _frame(s, store, warm_cameras=cams[:1])
    assert warm._warm_pairs is None and len(warm._warm) == 1
    for kw in (dict(camera=cams[0]), dict(timestep=0), dict(frames=1), dict(cameras=cams[:1])):
        with pytest.raises(ValueError, match="samples its camera, timestep and frame ids from its schedule"):
            fr.set_inputs(**kw)
    from gaussianavatars_b200.graph import GraphedFrame
    with pytest.raises(ValueError, match="cannot join a prefetching pair"):
        fr.prefetch_for(fr)
    plain = GraphedFrame(_model(), W, H, 0.7, 0.5, torch.zeros(3))
    for call in (lambda: plain.run_iterations(1), lambda: plain.set_cursor(0), lambda: plain.loss_history()):
        with pytest.raises(ValueError, match="schedule="):
            call()


def test_scheduled_run_is_bounded_on_the_host(cpu_schedule, no_device):
    S = cpu_schedule
    store = _store(n=3)
    s = S.ViewSchedule(_cams(3), frames=[0, 1, 2], order=[2, 0, 1, 1, 0])
    fr = _frame(s, store)
    assert fr.run_iterations(2, check=False) is None and fr.captures == 1 and fr.replays == 2
    fr.run()   # one iteration, check=False
    assert fr.replays == 3
    with pytest.raises(ValueError, match="3 more iterations could run past the schedule's 5"):
        fr.run_iterations(3, check=False)
    assert fr.replays == 3   # refused before anything ran
    fr.run_iterations(2, check=False)
    with pytest.raises(ValueError, match="could run past"):
        fr.run_iterations(1, check=False)
    with pytest.raises(ValueError, match=">= 0"):
        fr.run_iterations(-1)
    fr.set_cursor(4)
    assert fr.cursor.tolist() == [4] and fr.exhausted.tolist() == [0]
    fr.run_iterations(1, check=False)
    fr.set_cursor(0)
    fr.run_iterations(5, check=False)
    assert fr.replays == 11 and fr.captures == 1
    for bad in (-1, 6):
        with pytest.raises(IndexError, match=r"the cursor lies in \[0, 5\]"):
            fr.set_cursor(bad)


def test_graphed_eval_schedule_refusals(cpu_schedule, no_device):
    from gaussianavatars_b200.graph import GraphedEval
    S = cpu_schedule
    cams = _cams(3)
    store = _store(n=3)
    s = S.ViewSchedule(cams, frames=[0, 1, 2])
    with pytest.raises(ValueError, match="give schedule= and frames= together"):
        GraphedEval(_model(), W, H, torch.zeros(3), views=3, schedule=s)
    with pytest.raises(ValueError, match="give schedule= and frames= together"):
        GraphedEval(_model(), W, H, torch.zeros(3), views=3, frames=store)
    with pytest.raises(ValueError, match="score 3 rows, the table has 2"):
        GraphedEval(_model(), W, H, torch.zeros(3), views=2, schedule=s, frames=store)
    with pytest.raises(ValueError, match="the backgrounds must be equal"):
        GraphedEval(_model(), W, H, torch.ones(3), views=3, schedule=s, frames=store)
    with pytest.raises(ValueError, match="frame store holds 41x24"):
        GraphedEval(_model(), W, H, torch.zeros(3), views=3, schedule=s, frames=_store(w=W + 1))
    ev = GraphedEval(_model(), W, H, torch.zeros(3), views=4, schedule=s, frames=store)
    assert ev.frame_ids.shape == (1,) and ev.losses is None and ev.cursor.tolist() == [0]
    with pytest.raises(ValueError, match="set_inputs is refused"):
        ev.set_inputs(view=0)
    ev.cursor.fill_(2)
    ev.reset()
    assert ev.cursor.tolist() == [0] and torch.isnan(ev.table).all()
    plain = GraphedEval(_model(), W, H, torch.zeros(3), views=2)
    with pytest.raises(ValueError, match="run_all needs"):
        plain.run_all()
