"""-m gpu: one CUDA-graph replay as a whole training iteration (graph.GraphedFrame with optimizer= and
densify_stats=True): the densification-statistics launch against the reference's lines, the capturable Adam against
today's host-stepped Adam and against the reference's learning-rate schedule (tests/golden/make_golden_lr.py), and the
captured iteration against the same iteration run eagerly -- including re-capture after the eager densify_and_prune /
reset_opacity / oneupSHdegree, and an overflowing replay that must change nothing."""
import os

import numpy as np
import pytest
import torch

from tests import helpers as h

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD_LR = np.load(os.path.join(os.path.dirname(__file__), "golden", "lr_schedule.npz"))
STATS = ("xyz_gradient_accum", "denom", "max_radii2D")
ATTR = {"xyz": "_xyz", "rotation": "_rotation", "scaling": "_scaling", "opacity": "_opacity",
        "f_dc": "_features_dc", "f_rest": "_features_rest"}
LRS = {"xyz": 1.6e-4, "rotation": 1e-3, "scaling": 5e-3, "opacity": 5e-2, "f_dc": 2.5e-3, "f_rest": 1.25e-4}


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def _g():
    import gaussianavatars_b200 as g
    return g


def _ulps(a, b):
    """|a - b| in units in the last place, elementwise (float32, same sign or zero)."""
    return (a.contiguous().view(torch.int32).long() - b.contiguous().view(torch.int32).long()).abs()


def _grads_close(a, b):   # the check of test_gpu_sync_modes: gradients differ only by atomic summation order
    for x, y in zip(a, b):
        scale = float(y.abs().max()) + 1e-30
        assert float((x - y).abs().max()) <= 2e-5 * scale, "gradients differ beyond atomic-order noise"


# ---- 1. statistics ----------------------------------------------------------------------------------------------
def _reference_stats(m, vp_grad, radii):
    """train.py:197 and scene/gaussian_model.py:517-519, as the reference writes them."""
    vis = radii > 0
    m.max_radii2D[vis] = torch.max(m.max_radii2D[vis], radii[vis])
    m.xyz_gradient_accum[vis] += torch.norm(vp_grad[vis, :2], dim=-1, keepdim=True)
    m.denom[vis] += 1


def _stats_model(P):
    from types import SimpleNamespace
    return SimpleNamespace(xyz_gradient_accum=torch.zeros((P, 1), device=DEV), denom=torch.zeros((P, 1), device=DEV),
                           max_radii2D=torch.zeros((P,), device=DEV))


def _compare_stats(ours, ref, n_acc, what):
    assert torch.equal(ours.denom, ref.denom), what
    assert torch.equal(ours.max_radii2D, ref.max_radii2D), what
    d = _ulps(ours.xyz_gradient_accum, ref.xyz_gradient_accum)
    n_off = int((d > 0).sum())
    print(f"{what}: xyz_gradient_accum {'bitwise equal' if n_off == 0 else f'{n_off} entries off, max {int(d.max())} ulp'}"
          f" after {n_acc} accumulations")
    assert int(d.max()) <= n_acc, what


def test_densification_stats_match_the_reference_lines():
    g = _g()
    from types import SimpleNamespace
    gen = torch.Generator(device="cuda").manual_seed(4)
    P, K = 100_000, 6
    ours, ref = _stats_model(P), _stats_model(P)
    for k in range(K):
        radii = torch.randint(0, 60, (P,), device=DEV, generator=gen, dtype=torch.int32)
        radii[torch.rand(P, device=DEV, generator=gen) < 0.35] = 0
        grad = torch.randn(P, 3, device=DEV, generator=gen) * 10.0 ** (-2 - k)
        vp = SimpleNamespace(grad=grad)
        g.add_densification_stats(ours, vp, radii)
        _reference_stats(ref, grad, radii)
    _compare_stats(ours, ref, K, "synthetic P=100k")
    assert int((ours.denom > 0).sum()) > P // 2 and int((ours.denom == 0).sum()) > 0

    # one rendered frame's viewspace_points.grad and radii
    from gaussianavatars_b200.renderer import render
    sc = h.avatar_scene(P=15_000, W=400, H=304, seed=5)
    pc = _model(sc)
    pc.update_mesh_properties(sc["verts"].to(DEV))
    out = render(sc["cam"].to(DEV), pc, Pipe, sc["bg"].to(DEV))
    out["render"].backward(torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(1)).to(DEV))
    n = pc._xyz.shape[0]
    ours, ref = _stats_model(n), _stats_model(n)
    for _ in range(3):
        g.add_densification_stats(ours, out["viewspace_points"], out["radii"])
        _reference_stats(ref, out["viewspace_points"].grad, out["radii"])
    _compare_stats(ours, ref, 3, "rendered frame")
    assert int((out["radii"] == 0).sum()) > 0 and int((out["radii"] > 0).sum()) > 0
    with pytest.raises(ValueError, match="max_radii2D"):
        bad = _stats_model(n)
        bad.max_radii2D = torch.zeros((n + 1,), device=DEV)
        g.add_densification_stats(bad, out["viewspace_points"], out["radii"])


# ---- 2-4. capturable Adam ------------------------------------------------------------------------------------------
SHAPES = [(100_000, 3), (100_000, 1, 3), (100_000, 15, 3), (100_000, 1), (100_000, 3), (100_000, 4), (7, 6), (1, 3),
          (13, 100), (5,)]
LRS10 = [1.6e-4, 2.5e-3, 1.25e-4, 5e-2, 5e-3, 1e-3, 1e-3, 1e-6, 1e-3, 1e-2]


def _ten_groups(init, capturable):
    ps = [torch.nn.Parameter(t.clone()) for t in init]
    opt = _g().Adam([{"params": [p], "lr": lr, "name": str(i)} for i, (p, lr) in enumerate(zip(ps, LRS10))], lr=0.0,
                    eps=1e-15, capturable=capturable)
    return ps, opt


def _set_grads(flat, ps_list, skip_last):
    """Gradient views at a 4-byte (not 16-byte) aligned offset of one flat buffer, as the fused backward hands out."""
    for ps in ps_list:
        off = 1
        for i, a in enumerate(ps):
            if skip_last and i == len(ps) - 1:
                a.grad = None
                continue
            a.grad = flat[off:off + a.numel()].view_as(a)
            off += a.numel()


def _compare_adam(ours, theirs, opt_o, opt_t, what):
    """Moments bitwise; parameters bitwise except where device pow/exp/log rounds a per-step scalar differently from
    the host's (counted, at most 1 ulp)."""
    n_off = 0
    for a, b in zip(ours, theirs):
        d = _ulps(a.detach(), b.detach())
        n_off += int((d > 0).sum())
        assert int(d.max()) <= 1, what
        if a in opt_o.state:
            so, st = opt_o.state[a], opt_t.state[b]
            assert torch.equal(so["exp_avg"], st["exp_avg"]) and torch.equal(so["exp_avg_sq"], st["exp_avg_sq"]), what
            assert float(so["step"]) == float(st["step"]), what
    print(f"{what}: {n_off} parameter entries 1 ulp off")
    return n_off


def test_capturable_adam_matches_the_host_stepped_adam_and_torch_checkpoints():
    g = _g()
    gen = torch.Generator(device="cuda").manual_seed(11)
    init = [torch.randn(*s, device=DEV, generator=gen) for s in SHAPES]
    flat = torch.zeros(sum(t.numel() for t in init) + 1, device=DEV)
    ours, opt = _ten_groups(init, True)
    theirs, ref = _ten_groups(init, False)
    for step in range(4):
        flat.normal_(generator=gen)
        flat.mul_(10.0 ** (-step * 2))
        _set_grads(flat, [ours, theirs], skip_last=step == 0)
        opt.step()
        ref.step()
        assert _compare_adam(ours, theirs, opt, ref, f"step {step + 1}") == 0
    for a in ours:
        st = opt.state[a]["step"]
        assert st.device == a.device and st.dtype == torch.float32 and st.dim() == 0
    assert float(opt.state[ours[-1]]["step"]) == 3.0    # skipped at the first step, like torch

    # deep into training: the step counter is all that changes in the bias corrections
    total_off = 0
    for t in (17, 1000, 4321, 65_537, 300_000, 599_999, 600_000):
        for a, b in zip(ours, theirs):
            with torch.no_grad():
                a.copy_(b)
            so, st = opt.state[a], ref.state[b]
            so["exp_avg"].copy_(st["exp_avg"])
            so["exp_avg_sq"].copy_(st["exp_avg_sq"])
            so["step"].fill_(t - 1)
            st["step"] = torch.tensor(float(t - 1))
        flat.normal_(generator=gen)
        _set_grads(flat, [ours, theirs], skip_last=False)
        opt.step()
        ref.step()
        total_off += _compare_adam(ours, theirs, opt, ref, f"step {t}")
    print(f"sampled steps: {total_off} parameter entries 1 ulp off in total")

    # checkpoints: ours -> torch.optim.Adam(capturable=True) -> ours, with the step counters on the device throughout
    tp = [torch.nn.Parameter(a.detach().clone()) for a in ours]
    t_opt = torch.optim.Adam([{"params": [p], "lr": lr, "name": str(i)} for i, (p, lr) in enumerate(zip(tp, LRS10))],
                             lr=0.0, eps=1e-15, capturable=True)
    t_opt.load_state_dict(opt.state_dict())
    for p in tp:
        s = t_opt.state[p]["step"]
        assert s.device == p.device and s.dtype == torch.float32
        p.grad = torch.ones_like(p)
    t_opt.step()
    opt.load_state_dict(t_opt.state_dict())
    for a, p in zip(ours, tp):
        s = opt.state[a]["step"]
        assert s.device == a.device and s.dtype == torch.float32 and float(s) == float(t_opt.state[p]["step"])
        assert torch.equal(opt.state[a]["exp_avg"], t_opt.state[p]["exp_avg"])
        a.grad = torch.ones_like(a)
    opt.step()
    assert float(opt.state[ours[0]]["step"]) == 600_002.0


@pytest.mark.parametrize("name", ["default", "delayed"])
def test_scheduled_step_equals_a_host_step_at_the_reference_learning_rate(name):
    g = _g()
    lr_init, lr_final, delay_steps, delay_mult, max_steps = GOLD_LR[f"{name}_args"].tolist()
    sched = g.expon_lr_schedule(lr_init=lr_init, lr_final=lr_final, lr_delay_steps=int(delay_steps),
                                lr_delay_mult=delay_mult, max_steps=int(max_steps))
    gen = torch.Generator(device="cuda").manual_seed(2)
    p0 = torch.randn(50_000, 3, device=DEV, generator=gen)
    a = torch.nn.Parameter(p0.clone())
    b = torch.nn.Parameter(p0.clone())
    opt = g.Adam([{"params": [a], "lr": 0.0, "name": "xyz", "lr_schedule": sched}], lr=0.0, eps=1e-15, capturable=True)
    ref = g.Adam([{"params": [b], "lr": 0.0, "name": "xyz"}], lr=0.0, eps=1e-15)
    n_off = 0
    for it, lr in zip(GOLD_LR["iterations"].tolist(), GOLD_LR[f"{name}_lr"].tolist()):
        a.grad = torch.randn(p0.shape, device=DEV, generator=gen)
        b.grad = a.grad.clone()
        if a in opt.state:
            with torch.no_grad():
                a.copy_(b)
            opt.state[a]["exp_avg"].copy_(ref.state[b]["exp_avg"])
            opt.state[a]["exp_avg_sq"].copy_(ref.state[b]["exp_avg_sq"])
            opt.state[a]["step"].fill_(it - 1)
            ref.state[b]["step"] = torch.tensor(float(it - 1))
        ref.param_groups[0]["lr"] = lr          # what update_learning_rate(iteration) writes
        opt.step()
        ref.step()
        n_off += _compare_adam([a], [b], opt, ref, f"{name} iteration {it}")
        assert float(opt.state[a]["step"]) == it
    print(f"{name}: {n_off} entries 1 ulp off over {len(GOLD_LR['iterations'])} iterations")


def test_adam_step_captured_in_a_cuda_graph_equals_eager_steps():
    g = _g()
    gen = torch.Generator(device="cuda").manual_seed(5)
    init = [torch.randn(*s, device=DEV, generator=gen) for s in SHAPES]
    ours, opt = _ten_groups(init, True)
    eager, opt_e = _ten_groups(init, True)
    host, opt_h = _ten_groups(init, False)
    static = [torch.zeros_like(p) for p in ours]
    for p, s in zip(ours, static):
        p.grad = s
    opt.init_state()
    before = [p.detach().clone() for p in ours]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    torch.cuda.synchronize()
    assert all(torch.equal(p, q) for p, q in zip(ours, before)), "capture changed a parameter"
    assert all(float(opt.state[p]["step"]) == 0.0 for p in ours)
    for k in range(5):
        grads = [torch.randn(p.shape, device=DEV, generator=gen) * 10.0 ** -k for p in ours]
        for s, gr in zip(static, grads):
            s.copy_(gr)
        graph.replay()
        for pe, ph, gr in zip(eager, host, grads):
            pe.grad, ph.grad = gr.clone(), gr.clone()
        opt_e.step()
        opt_h.step()
        torch.cuda.synchronize()
        for a, b in zip(ours, eager):
            assert torch.equal(a, b), f"replay {k}: parameter differs from the eager capturable step"
            for key in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(opt.state[a][key], opt_e.state[b][key]), (k, key)
        _compare_adam(ours, host, opt, opt_h, f"replay {k} vs host-stepped Adam")


# ---- 5-7. the whole iteration in one graph --------------------------------------------------------------------------
def _model(sc, sh_degree=3):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians

    pc = MeshBoundGaussians(sc["params"], sh_degree, sc["verts"], sc["faces"], pose_fn=syn.pose_mesh, device=DEV,
                            requires_grad=True)
    return pc


def _trainable(sc):
    """A mesh-bound model carrying what train.py's GaussianModel carries: an optimizer with the reference's named
    groups (xyz on the exponential schedule), the densification statistics, percent_dense and binding_counter."""
    g = _g()
    pc = _model(sc)
    for n, attr in ATTR.items():
        setattr(pc, attr, torch.nn.Parameter(getattr(pc, attr).detach().clone()))
    groups = []
    for n, attr in ATTR.items():
        gr = {"params": [getattr(pc, attr)], "lr": LRS[n], "name": n}
        if n == "xyz":
            gr["lr_schedule"] = g.expon_lr_schedule(lr_init=5e-3, lr_final=5e-5, lr_delay_mult=0.01, max_steps=600_000)
        groups.append(gr)
    pc.optimizer = g.Adam(groups, lr=0.0, eps=1e-15, capturable=True)
    P = pc._xyz.shape[0]
    pc.xyz_gradient_accum = torch.zeros((P, 1), device=DEV)
    pc.denom = torch.zeros((P, 1), device=DEV)
    pc.max_radii2D = torch.zeros((P,), device=DEV)
    pc.percent_dense = 0.01
    pc.binding_counter = torch.bincount(pc.binding.long(), minlength=sc["faces"].shape[0]).to(torch.int32)
    return pc


def _snapshot(pc):
    opt = pc.optimizer
    snap = {"params": [p.detach().clone() for p in pc.parameters()],
            "stats": [getattr(pc, n).clone() for n in STATS], "state": []}
    for p in pc.parameters():
        st = opt.state.get(p, {})
        snap["state"].append({k: v.clone() for k, v in st.items()})
    return snap


def _assert_state_equal(pc, snap, what):
    opt = pc.optimizer
    for p, q in zip(pc.parameters(), snap["params"]):
        assert torch.equal(p.detach(), q), f"{what}: parameter changed"
    for n, s in zip(STATS, snap["stats"]):
        assert torch.equal(getattr(pc, n), s), f"{what}: {n} changed"
    for p, st in zip(pc.parameters(), snap["state"]):
        for k, v in st.items():
            assert torch.equal(opt.state[p][k], v), f"{what}: {k} changed"


def _expected_after_step(pc, snap, grads, vp_grad, radii):
    """The eager iteration on a copy of the pre-replay state with the replay's own gradients: add_densification_stats
    + capturable Adam.step()."""
    from types import SimpleNamespace
    g = _g()
    ps = [torch.nn.Parameter(q.clone()) for q in snap["params"]]
    groups = []
    for gr, p in zip(pc.optimizer.param_groups, ps):
        groups.append({k: v for k, v in gr.items() if k != "params"} | {"params": [p]})
    opt = g.Adam(groups, lr=0.0, eps=1e-15, capturable=True)
    for p, st in zip(ps, snap["state"]):
        if st:
            opt.state[p] = {k: v.clone() for k, v in st.items()}
    for p, gr in zip(ps, grads):
        p.grad = gr.clone()
    m = SimpleNamespace(**{n: s.clone() for n, s in zip(STATS, snap["stats"])})
    g.add_densification_stats(m, SimpleNamespace(grad=vp_grad.clone()), radii.clone())
    opt.step()
    return ps, opt, m


def _check_replay(fr, pc, snap, eager_ref, what):
    img_ref, grads_ref = eager_ref
    assert torch.equal(fr.image, img_ref), f"{what}: image differs from the eager frame"
    grads = [p.grad for p in pc.parameters()]
    _grads_close(grads, grads_ref)
    ps, opt, m = _expected_after_step(pc, snap, grads, fr.viewspace_points.grad, fr.radii)
    for p, q in zip(pc.parameters(), ps):
        assert torch.equal(p.detach(), q.detach()), f"{what}: parameter differs from the eager step"
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(pc.optimizer.state[p][k], opt.state[q][k]), f"{what}: {k} differs"
    for n in STATS:
        assert torch.equal(getattr(pc, n), getattr(m, n)), f"{what}: {n} differs"


def _eager_frame(sc, snap, verts, cam, gt, active_sh_degree):
    """Image and parameter gradients of the eager frame (render + photometric loss + regularisers + backward) on the
    pre-replay parameters."""
    g = _g()
    from gaussianavatars_b200.renderer import render
    pc_e = _model(sc)
    P = snap["params"][0].shape[0]
    for attr, q in zip(ATTR.values(), snap["params"]):
        setattr(pc_e, attr, q.clone().requires_grad_(True))
    if pc_e.binding.shape[0] != P:
        raise AssertionError("eager model must follow the densified binding")
    pc_e.active_sh_degree = active_sh_degree
    v = verts.to(DEV).clone().requires_grad_(True)
    pc_e.update_mesh_properties(v)
    out = render(cam.to(DEV), pc_e, Pipe, sc["bg"].to(DEV))
    loss = g.photometric_loss(out["render"], gt, 0.2)
    lx, ls = g.binding_regularizers(pc_e._xyz, pc_e._scaling, out["radii"], pc_e.binding, pc_e.face_scaling)
    (loss + lx + ls).backward()
    torch.cuda.synchronize()
    return out["render"].detach().clone(), [p.grad.clone() for p in pc_e.parameters()]


def _scene():
    sc = h.avatar_scene(P=15_000, W=400, H=304, seed=5)
    gt = torch.randint(0, 256, (3, sc["H"], sc["W"]), generator=torch.Generator().manual_seed(7),
                       dtype=torch.uint8).to(DEV)
    return sc, gt


def _frame(pc, sc, gt, **kw):
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    cam = sc["cam"]
    fr = GraphedFrame(pc, sc["W"], sc["H"], cam.FoVx, cam.FoVy, sc["bg"], loss="photometric", regularizers={},
                      optimizer=pc.optimizer, densify_stats=True, **kw)
    fr.set_inputs(camera=camera_block(cam), verts=sc["verts"].to(DEV), gt_u8=gt)
    return fr


def _replay_and_check(fr, pc, sc, gt, verts, what, check=True):
    # the eager model mirrors the current binding (densify_and_prune replaces it)
    sc_now = dict(sc)
    sc_now["params"] = dict(sc["params"])
    sc_now["params"]["binding"] = pc.binding
    snap = _snapshot(pc)
    ref = _eager_frame(sc_now, snap, verts, sc["cam"], gt, pc.active_sh_degree)
    fr.set_inputs(verts=verts.to(DEV))
    fr.run(check=check)
    torch.cuda.synchronize()
    _check_replay(fr, pc, snap, ref, what)


def test_whole_training_iteration_in_one_graph_equals_the_eager_iteration():
    from gaussianavatars_b200 import synthetic as syn
    sc, gt = _scene()
    pc = _trainable(sc)
    fr = _frame(pc, sc, gt)
    pc.optimizer.init_state()
    snap = _snapshot(pc)
    fr.capture()
    torch.cuda.synchronize()
    _assert_state_equal(pc, snap, "capture")
    verts2 = syn.pose_mesh(sc["verts"], 9)
    for i, verts in enumerate((sc["verts"], verts2, sc["verts"])):
        _replay_and_check(fr, pc, sc, gt, verts, f"replay {i}")
        assert fr.captures == 1
    assert float(pc.optimizer.state[pc._xyz]["step"]) == 3.0
    assert float(pc.denom.max()) == 3.0 and float(pc.max_radii2D.max()) > 0


def test_replaced_state_is_recaptured():
    import gaussianavatars_b200 as g
    sc, gt = _scene()
    pc = _trainable(sc)
    pc.active_sh_degree = 2
    fr = _frame(pc, sc, gt)
    fr.capture()
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "first replay")
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "second replay")
    assert fr.captures == 1

    # reset_opacity (scene/gaussian_model.py:277-280 + replace_tensor_to_optimizer :334-347)
    with torch.no_grad():
        op = torch.sigmoid(pc._opacity)
        new = torch.logit(torch.min(op, torch.ones_like(op) * 0.01))
    gr = next(gr for gr in pc.optimizer.param_groups if gr["name"] == "opacity")
    st = pc.optimizer.state.pop(gr["params"][0])
    st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(new), torch.zeros_like(new)
    gr["params"][0] = torch.nn.Parameter(new.requires_grad_(True))
    pc.optimizer.state[gr["params"][0]] = st
    pc._opacity = gr["params"][0]
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "after reset_opacity")
    assert fr.captures == 2

    # densify_and_prune: new parameters, moments, statistics and P
    P0 = pc._xyz.shape[0]
    grads = pc.xyz_gradient_accum / pc.denom
    thr = float(torch.nan_to_num(grads, 0.0).quantile(0.9))
    info = g.densify_and_prune(pc, thr, 0.005, 1.0, None, generator=torch.Generator(DEV).manual_seed(3))
    assert info["P_out"] != P0 and pc._xyz.shape[0] == info["P_out"]
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "after densify_and_prune")
    assert fr.captures == 3

    # oneupSHdegree
    pc.active_sh_degree += 1
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "after oneupSHdegree")
    assert fr.captures == 4
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "steady")
    assert fr.captures == 4


def test_an_overflowing_replay_applies_no_step():
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.graph import camera_block
    sc, gt = _scene()
    pc = _trainable(sc)
    # the frame's own camera and, last, another one: the step after re-capture must train on the frame's camera
    other = syn.orbit_camera(sc["W"], sc["H"], r=1.0, fovy_deg=20.0, azimuth_deg=25.0)
    warm = [camera_block(sc["cam"]), camera_block(other)]
    fr = _frame(pc, sc, gt, warm_cameras=warm)
    pc.optimizer.init_state()
    snap = _snapshot(pc)
    fr.capture(capacity=4096)            # far below what the frame needs
    fr.run(check=False)
    assert fr.overflowed(wait=True), "an overflowing replay was not flagged"
    _assert_state_equal(pc, snap, "overflowing replay")
    _replay_and_check(fr, pc, sc, gt, sc["verts"], "regrown replay", check=True)
    assert fr.captures == 2 and not fr.overflowed(wait=True)
    assert float(pc.optimizer.state[pc._xyz]["step"]) == 1.0
