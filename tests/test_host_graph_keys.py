"""CPU: what makes a captured frame stale -- the changes between replays after which GraphedFrame (the training step)
and GraphedRender (the playback frame) re-capture on their next run(), and those after which they must not.  The
capture itself is stubbed out (no device, no graph): run() compares what the last capture baked in with the model as
it is now, and that comparison only reads addresses, shapes, versions and host values."""
import contextlib
from types import SimpleNamespace

import pytest
import torch

PARAMS = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
POSED = ("expr", "rotation", "neck_pose", "jaw_pose", "eyes_pose", "translation")
W, H = 64, 48


class _NoGraph:
    def replay(self):
        pass


@pytest.fixture(autouse=True)
def _no_device(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _NoGraph)
    monkeypatch.setattr(torch.cuda, "graph", lambda g: contextlib.nullcontext())


def _model(flame=False, P=4):
    pc = SimpleNamespace(active_sh_degree=0, binding=torch.zeros(P, dtype=torch.int32),
                         face_center=torch.zeros(2, 3), face_orien_mat=torch.zeros(2, 3, 3),
                         face_scaling=torch.ones(2, 1), xyz_gradient_accum=torch.zeros(P, 1),
                         denom=torch.zeros(P, 1), max_radii2D=torch.zeros(P))
    for n in PARAMS:
        setattr(pc, n, torch.nn.Parameter(torch.zeros(P, 3)))
    pc.parameters = lambda: [getattr(pc, n) for n in PARAMS]
    if flame:
        pc.flame = object()
        pc.flame_param = {"shape": torch.zeros(10), "static_offset": torch.zeros(1, 5, 3)}
        pc.flame_param.update({k: torch.zeros(6, 3, requires_grad=True) for k in POSED})
    else:
        pc.verts_rest = torch.zeros(5, 3)
    return pc


def _stubbed(frame):
    frame._learn_capacity = lambda: (0, (0, 0))
    frame._body = lambda *a, **k: None
    return frame


def _train(flame=False, full=False):
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.graph import GraphedFrame

    pc = _model(flame)
    opt = g.Adam([{"params": [getattr(pc, n)], "lr": 1e-3, "name": n} for n in PARAMS], eps=1e-15,
                 capturable=True) if full else None
    return _stubbed(GraphedFrame(pc, W, H, 0.7, 0.5, torch.zeros(3), optimizer=opt, densify_stats=full))


def _render(flame=False, mesh_update=True):
    from gaussianavatars_b200.graph import GraphedRender

    return _stubbed(GraphedRender(_model(flame), W, H, torch.zeros(3), mesh_update=mesh_update))


FRAMES = {
    "train": lambda: _train(),                                 # no optimizer, no statistics, no FLAME head
    "train_full": lambda: _train(full=True),                   # capturable Adam + densification statistics
    "train_flame": lambda: _train(flame=True),
    "render": lambda: _render(),
    "render_flame": lambda: _render(flame=True),
    "render_fixed_mesh": lambda: _render(mesh_update=False),   # renders the face frame the model holds
}


def _densify(fr):
    P = fr.pc._xyz.shape[0] + 1
    for n in PARAMS:
        setattr(fr.pc, n, torch.nn.Parameter(torch.zeros(P, 3)))


def _edit_param(fr):
    with torch.no_grad():
        fr.pc._xyz.add_(1.0)


def _oneup_sh(fr):
    fr.pc.active_sh_degree += 1


def _new_binding(fr):
    fr.pc.binding = fr.pc.binding.clone()


def _new_face_frame(fr):
    fr.pc.face_center = fr.pc.face_center.clone()


def _new_statistic(fr):
    fr.pc.denom = torch.zeros_like(fr.pc.denom)


def _host_lr(fr):
    fr.optimizer.param_groups[0]["lr"] *= 0.5


def _new_moment(fr):
    st = fr.optimizer.state[fr.pc._xyz]
    st["exp_avg"] = torch.zeros_like(st["exp_avg"])


def _flame_requires_grad(fr):
    fr.pc.flame_param["expr"].requires_grad_(False)


def _edit_shape(fr):
    fr.pc.flame_param["shape"].add_(1.0)


def _edit_expr(fr):     # a viewer's slider
    with torch.no_grad():
        fr.pc.flame_param["expr"][2].add_(1.0)


def _new_flame_tensor(fr):
    fr.pc.flame_param["jaw_pose"] = fr.pc.flame_param["jaw_pose"].detach().clone().requires_grad_(True)


def _timestep(fr):
    fr.set_inputs(timestep=3)


def _camera_same_size(fr):
    from gaussianavatars_b200 import synthetic as syn
    fr.set_inputs(camera=syn.orbit_camera(W, H, azimuth_deg=30.0))


def _camera_other_size(fr):
    from gaussianavatars_b200 import synthetic as syn
    fr.set_inputs(camera=syn.orbit_camera(W + 16, H + 12))


def _scaling_modifier(fr):
    fr.scaling_modifier = 0.5


def _background(fr):
    fr.set_inputs(bg=torch.ones(3))


CASES = [   # (frame, change between replays, re-captures)
    ("train", _densify, False), ("train", _oneup_sh, False), ("train", _new_binding, False),
    ("train", _edit_param, False), ("train", _new_face_frame, False), ("train", _new_statistic, False),
    ("train", _camera_same_size, False),
    ("train_full", _densify, True), ("train_full", _oneup_sh, True), ("train_full", _new_binding, True),
    ("train_full", _new_statistic, True), ("train_full", _host_lr, True), ("train_full", _new_moment, True),
    ("train_full", _edit_param, False), ("train_full", _new_face_frame, False),
    ("train_full", _camera_same_size, False),
    ("train_flame", _densify, True), ("train_flame", _oneup_sh, True), ("train_flame", _new_binding, True),
    ("train_flame", _flame_requires_grad, True), ("train_flame", _edit_shape, True),
    ("train_flame", _new_flame_tensor, True), ("train_flame", _edit_expr, False), ("train_flame", _timestep, False),
    ("train_flame", _new_face_frame, False), ("train_flame", _new_statistic, False),
    ("train_flame", _edit_param, False),
    ("render", _densify, True), ("render", _oneup_sh, True), ("render", _new_binding, True),
    ("render", _camera_other_size, True), ("render", _scaling_modifier, True), ("render", _camera_same_size, False),
    ("render", _background, False), ("render", _edit_param, False), ("render", _new_face_frame, False),
    ("render", _new_statistic, False),
    ("render_flame", _densify, True), ("render_flame", _edit_shape, True), ("render_flame", _new_flame_tensor, True),
    ("render_flame", _flame_requires_grad, False), ("render_flame", _edit_expr, False),
    ("render_flame", _timestep, False), ("render_flame", _new_face_frame, False),
    ("render_fixed_mesh", _new_face_frame, True), ("render_fixed_mesh", _new_binding, True),
    ("render_fixed_mesh", _edit_param, False), ("render_fixed_mesh", _camera_same_size, False),
]


@pytest.mark.parametrize("kind, change, recaptures", CASES,
                         ids=[f"{k}-{c.__name__.lstrip('_')}" for k, c, _ in CASES])
def test_a_change_between_replays_recaptures_exactly_when_the_capture_baked_it_in(kind, change, recaptures):
    fr = FRAMES[kind]()
    fr.run()
    fr.run()
    assert (fr.captures, fr.replays) == (1, 2)
    change(fr)
    fr.run()
    assert fr.captures == (2 if recaptures else 1)
    fr.run()
    assert fr.captures == (2 if recaptures else 1), "a re-capture must remember the new state"
