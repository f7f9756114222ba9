"""CPU: what makes a GraphedEval stale -- the evaluation graph re-captures after exactly the changes that re-capture a
GraphedRender (P, active_sh_degree, the parameter addresses, the image size), and never for the inputs of a view: its
camera, timestep, ground truth, table row and background.  The capture itself is stubbed out (no device, no graph), as
in test_host_graph_keys.py."""
import pytest
import torch

from tests.test_host_graph_keys import PARAMS, W, H, _model, _no_device, _stubbed  # noqa: F401  (autouse fixture)


def _eval(flame=False, source="float"):
    from gaussianavatars_b200.graph import GraphedEval

    return _stubbed(GraphedEval(_model(flame), W, H, torch.zeros(3), views=8, source=source))


def _camera_same_size(ev):
    from gaussianavatars_b200 import synthetic as syn
    ev.set_inputs(camera=syn.orbit_camera(W, H, azimuth_deg=30.0, fovy_deg=35.0))


def _camera_other_size(ev):
    from gaussianavatars_b200 import synthetic as syn
    ev.set_inputs(camera=syn.orbit_camera(W + 16, H + 12), gt_u8=torch.ones((3, H + 12, W + 16), dtype=torch.uint8))


def _timestep(ev):
    ev.set_inputs(timestep=3)


def _gt(ev):
    ev.set_inputs(gt_u8=torch.full((3, H, W), 7, dtype=torch.uint8))


def _view(ev):
    ev.set_inputs(view=5)


def _background(ev):
    ev.set_inputs(bg=torch.ones(3))


def _reset(ev):
    ev.reset()


def _densify(ev):
    P = ev.pc._xyz.shape[0] + 1
    for n in PARAMS:
        setattr(ev.pc, n, torch.nn.Parameter(torch.zeros(P, 3)))


def _oneup_sh(ev):
    ev.pc.active_sh_degree += 1


def _new_param_tensor(ev):   # same P, another address (a checkpoint loaded into fresh tensors)
    ev.pc._opacity = torch.nn.Parameter(ev.pc._opacity.detach().clone())


def _edit_param(ev):
    with torch.no_grad():
        ev.pc._xyz.add_(1.0)


CASES = [   # (change between replays, re-captures)
    (_camera_same_size, False), (_timestep, False), (_gt, False), (_view, False), (_background, False),
    (_reset, False), (_edit_param, False),
    (_densify, True), (_oneup_sh, True), (_new_param_tensor, True), (_camera_other_size, True),
]


@pytest.mark.parametrize("source", ["float", "u8"])
@pytest.mark.parametrize("change, recaptures", CASES, ids=[c.__name__.lstrip("_") for c, _ in CASES])
def test_a_view_never_recaptures_and_the_model_does(change, recaptures, source):
    ev = _eval(flame=change is _timestep, source=source)
    ev.run()
    ev.run()
    assert (ev.captures, ev.replays) == (1, 2)
    change(ev)
    ev.run()
    assert ev.captures == (2 if recaptures else 1)
    ev.run()
    assert ev.captures == (2 if recaptures else 1), "a re-capture must remember the new state"


def test_the_key_is_the_playback_key():
    from gaussianavatars_b200.graph import GraphedRender
    ev = _eval()
    view = _stubbed(GraphedRender(ev.pc, W, H, torch.zeros(3), outputs="float"))
    assert ev._state_key() == view._state_key()
