"""-m gpu: the backward blend on the walk scenes (tests/walk_scenes.py), whose warps between them take every branch of
the walk that tests/test_oracle_walk.py's census lists, under the light-only schedule (K = 4 on every tile) and
HEAVY_BWD = 32 (K = 2 on every tile of 32 or more entries), with the colour backward and with the depth plane
(the backward's tenth row, dL/dz), single-view here and K-view in tests/test_gpu_multiview_adversarial.py.

Colour: radii and the sorted stream bit-exact; image, final_T and every input gradient against the C oracle and against float64 autograd of the dense model under the
explained gates (helpers.assert_image_explained / assert_grad_explained): outside the knife set of
adversarial_scenes.knife_edges, no entry beyond the tolerance.  Depth plane: the alpha and depth planes against the
oracle, dL/d_xyz and dL/dmeans2D of <alpha, ga> + <depth, gd> against float64, under the same gates
(test_gpu_depth_alpha.planes_against_the_oracle_and_float64).  Each comparison prints the size of its knife set."""
import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import helpers as h
from tests import walk_scenes as WS
from tests.test_gpu_adversarial import _run

pytestmark = pytest.mark.gpu

SCHEDULES = ["light", "bwd32"]


@pytest.fixture(params=SCHEDULES)
def schedule(request):
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import rasterizer as R

    knobs = {N.TUNE_TILE_SORT: 0, N.TUNE_DEPTH_SORT: 1}
    if request.param == "bwd32":
        knobs[N.TUNE_HEAVY_BWD] = 32
    prev = {k: N.tune(k, v) for k, v in knobs.items()}
    prev_exact = R._EXACT_BINNING
    R.set_exact_binning(True)
    R.keep_last_state(True)
    yield request.param
    R.set_exact_binning(prev_exact)
    for k, v in prev.items():
        N.tune(k, v)


_REF = {}


def _reference(name):
    if name not in _REF:
        from tests.test_oracle_adversarial import dense_image_and_grads

        sc = WS.build(name)
        st = h.oracle_forward(sc)
        gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(7))
        g = h.oracle_backward(sc, st, gout.numpy())
        img64, g64 = dense_image_and_grads(sc, st, seed=7)
        ke = A.knife_edges(st)
        print(f"[knife] walk {name}: {ke['pairs']} pairs, {int(ke['pixels'].sum())} pixels, "
              f"{int(ke['splats'].sum())}/{st.P} splats")
        _REF[name] = dict(sc=sc, st=st, gout=gout, g=g, img64=img64, g64=g64, ke=ke)
    return _REF[name]


@pytest.mark.parametrize("name", list(WS.WALK))
def test_backward_walk(name, schedule):
    ref = _reference(name)
    sc, st, ke = ref["sc"], ref["st"], ref["ke"]
    what = f"walk {name} [{schedule}]"
    out = _run(sc, (0, 1, True, schedule), ref["gout"])
    assert np.array_equal(out["radii"], st.radii), f"{what}: radii differ from the oracle"
    assert out["n"] == st.N, f"{what}: {out['n']} instances, oracle {st.N}"
    assert np.array_equal(out["keys"], st.keys_sorted), f"{what}: sorted tile|depth keys not bit-exact"
    assert np.array_equal(out["vals"], st.vals_sorted), f"{what}: sorted splat ids not bit-exact"
    assert np.array_equal(out["ranges"], st.ranges), f"{what}: tile ranges differ"
    img = out["img"].cpu().numpy()
    h.assert_image_explained(img, st.out_color, ke["pixels"], f"{what}: image")
    h.assert_image_explained(out["T"], np.broadcast_to(st.final_T, out["T"].shape), ke["pixels"], f"{what}: final_T")
    h.assert_image_explained(img, ref["img64"], ke["pixels"], f"{what}: image vs float64")
    for k, g in out["grads"].items():
        h.assert_grad_explained(g, ref["g"][k], A.affected(ke, k), f"{name} dL/d{k}")
        h.assert_grad_explained(g, ref["g64"][k], A.affected(ke, k), f"{name} dL/d{k} vs float64")


@pytest.mark.parametrize("name", list(WS.WALK))
def test_backward_walk_depth_plane(name, schedule):
    from tests.test_gpu_depth_alpha import planes_against_the_oracle_and_float64

    planes_against_the_oracle_and_float64(WS.build(name), f"walk {name} depth plane [{schedule}]")
