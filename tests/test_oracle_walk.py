"""CPU: the walk scenes (tests/walk_scenes.py) reach every branch of the backward blend's walk, and
adversarial_scenes.knife_edges finds the threshold decisions that can flip, and only those.

A scene change that stops reaching an item of walk_scenes.WANTED fails here rather than silently weakening
tests/test_gpu_backward_walk.py."""
import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import helpers as h
from tests import walk_scenes as WS
from tests.test_oracle_adversarial import dense_image_and_grads

_ST = {}


def _state(name):
    if name not in _ST:
        sc = WS.build(name)
        _ST[name] = (sc, h.oracle_forward(sc))
    return _ST[name]


def test_walk_scenes_reach_every_branch_of_the_walk():
    got = set()
    for name in WS.WALK:
        _, st = _state(name)
        lens = st.ranges[:, 1].astype(np.int64) - st.ranges[:, 0]
        assert list(lens) == WS.WALK[name][0], f"{name}: tile lists are not the scene's own splats"
        for depth, heavy in WS.RUNS:
            got |= {(depth,) + item for item in WS.reached(WS.census(st, heavy))}
    missing = sorted(WS.WANTED - got, key=str)
    assert not missing, f"walk items no scene reaches: {missing}"


@pytest.mark.parametrize("name", list(WS.WALK))
def test_walk_rig_interleaves_views_and_walks_both_k(name):
    """The K-view frame of tests/test_gpu_multiview_adversarial.py::test_walk_scenes_six_views: its global tile order
    interleaves the views, and its views' warps walk under K = 2 and K = 4."""
    from tests import bound_rigs as B
    from tests import train_step_oracle as T
    bound = B.bind(WS.build(name))
    act, _, _ = B.activate(bound)
    act = {k: v.detach() for k, v in act.items()}
    fl = dict(sh_degree=bound["sh_degree"], bg=bound["bg"].numpy())
    sts = [T.oracle_forward_on(act["means3D"], act["opacities"], cam, bound["W"], bound["H"], fl, act["shs"],
                               scales=act["scales"], rotations=act["rotations"]) if B.valid(k) else None
           for k, cam in enumerate(B.rig(bound, 6))]
    assert WS.views_interleave(sts), f"{name}: the views' tiles do not interleave in the global order"
    ks = {r["K"] for st in sts if st is not None for r in WS.census(st, 32)}
    assert ks == {2, 4}, f"{name}: the K-view walk under HEAVY_BWD = 32 takes K in {ks} only"


@pytest.mark.parametrize("name", list(WS.WALK) + ["saturating_stack", "faint"])
def test_knife_edges_restate_the_oracle_walk(name):
    """The walk knife_edges restates is the oracle's: n_contrib exactly, final_T to the ulp of the oracle's expf."""
    st = _state(name)[1] if name in WS.WALK else h.oracle_forward(A.build(name))
    ke = A.knife_edges(st)
    assert np.array_equal(ke["n_contrib"], st.n_contrib.astype(np.int64))
    assert np.abs(ke["final_T"] - st.final_T).max() <= 4 * np.spacing(np.float32(1))


@pytest.mark.parametrize("name", list(WS.WALK))
def test_oracle_equals_float64_on_walk_scenes(name):
    sc, st = _state(name)
    ke = A.knife_edges(st)
    print(f"[knife] walk {name}: {ke['pairs']} pairs, {int(ke['pixels'].sum())} pixels, "
          f"{int(ke['splats'].sum())}/{st.P} splats")
    img, g64 = dense_image_and_grads(sc, st, seed=3)
    h.assert_image_explained(st.out_color, img, ke["pixels"], "oracle image vs float64", tol=5e-6, cap=5e-6)
    gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(3))
    g = h.oracle_backward(sc, st, gout.numpy())
    for k, ref in g64.items():
        h.assert_grad_explained(g[k], ref, A.affected(ke, k), f"walk {name} dL/d{k}", knife_allowed=0)


# ---- knife_edges on scenes built on and clear of each threshold -------------------------------------------------------
def _pixel_scene(opac, offsets=None, sigma=1.2, W=16, H=16):
    """Splats centred exactly on pixel (7, 7) (or on `offsets` in pixels from it) at increasing depth."""
    n = len(opac)
    f = A.default_focal(W, H)
    cam = A.camera(W, H, f)
    off = np.zeros((n, 2)) if offsets is None else np.asarray(offsets, np.float64)
    z = 2.0 + 0.01 * np.arange(n)
    xyz = A.unproject(cam, W, H, 7.0 + off[:, 0], 7.0 + off[:, 1], z, exact=True)
    s = sigma * z / f
    rot = np.tile([1.0, 0, 0, 0], (n, 1))
    return A._scene(cam, W, H, xyz, np.stack([s, s, s], 1), rot, opac, np.zeros((n, 1, 3)) + 0.2, 0)


def _alpha_at(st, splat, x, y):
    co = st.conic_opacity[splat]
    dx, dy = st.xy[splat, 0] - np.float32(x), st.xy[splat, 1] - np.float32(y)
    return np.float32(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy


@pytest.mark.parametrize("rel,knife", [(0.0, True), (3e-7, True), (-3e-7, True), (1e-4, False), (-1e-4, False)])
def test_alpha_threshold_knife(rel, knife):
    """One splat whose alpha at the pixel beside its centre is 1/255 (1 + rel): within the bound it is a knife pair
    there; at its exact centre alpha = opacity bit for bit on both sides and nothing is a knife."""
    sc = _pixel_scene([0.5])
    st = h.oracle_forward(sc)
    power = _alpha_at(st, 0, 8, 7)
    o = np.float32(float(A.ALPHA_MIN) * (1 + rel) / np.exp(np.float64(power)))
    st = h.oracle_forward(dict(sc, opacities=torch.tensor([[o]])))
    ke = A.knife_edges(st)
    assert bool(ke["pixels"][7, 8]) == knife and (bool(ke["splats"][0]) or not knife)
    assert not ke["pixels"][7, 7]


def test_exact_centre_on_the_alpha_threshold_is_not_a_knife():
    """Opacity float32(1/255) and one ulp below at their exact centres: the decision is exact, not a knife."""
    thr = A.ALPHA_MIN
    sc = _pixel_scene([thr, np.nextafter(thr, np.float32(0))], offsets=[(0, 0), (0, 0)], sigma=0.3)
    st = h.oracle_forward(sc)
    ke = A.knife_edges(st)
    assert not ke["pixels"][7, 7] and st.n_contrib[7, 7] == 1


def _stop_scene(side):
    """Splats of alpha 0.99 and 0.9 on the pixel centre (7, 7), a third half a pixel off it whose alpha there puts T
    nearest 1e-4 on `side` (-1: below, the walk stops on it; 1: at or above), and a fourth behind."""
    sc = _pixel_scene([0.995, 0.9, 0.9, 0.5], offsets=[(0, 0), (0, 0), (0.5, 0), (0, 0)], sigma=1.2)
    st = h.oracle_forward(sc)
    g3 = np.float32(np.exp(np.float64(_alpha_at(st, 2, 7, 7))))
    t2 = (np.float32(1) - np.float32(0.99)) * (np.float32(1) - np.float32(0.9))
    o = np.float32((1 - 1e-4 / float(t2)) / float(g3))
    cand = [o]
    for step in (np.float32(0), np.float32(1)):
        c = o
        for _ in range(64):
            c = np.nextafter(c, step)
            cand.append(c)
    cand = np.array(cand, np.float32)
    t = t2 * (np.float32(1) - np.minimum(np.float32(0.99), cand * g3))
    ok = (t < A.T_STOP) if side < 0 else (t >= A.T_STOP)
    o3 = cand[ok][np.argmin(np.abs(t[ok].astype(np.float64) - float(A.T_STOP)))]
    return dict(sc, opacities=torch.tensor([[0.995], [0.9], [float(o3)], [0.5]]))


@pytest.mark.parametrize("side", [-1, 1])
def test_stop_threshold_knife(side):
    """T lands within the bound of 1e-4 at the third splat (stopping there or not): the pixel is a knife and every
    splat of it, the one behind included, is affected.  On the exact centre T is exact on both sides: two splats of
    alpha 0.99 end the walk without a knife, and with a clear margin nothing is a knife either."""
    st = h.oracle_forward(_stop_scene(side))
    assert st.n_contrib[7, 7] == (2 if side < 0 else 3)
    ke = A.knife_edges(st)
    assert ke["pixels"][7, 7] and ke["splats"].all()
    for opac in ([0.995, 0.995, 0.5], [0.995, 0.9, 0.5]):
        clear = h.oracle_forward(_pixel_scene(opac, sigma=0.3))
        ke = A.knife_edges(clear)
        assert not ke["pixels"].any() and not ke["splats"].any()


@pytest.mark.parametrize("b_scale,knife", [(1 + 1e-7, True), (1 - 1e-7, True), (0.9, False)])
def test_power_threshold_knife(b_scale, knife):
    """A conic with B = b_scale sqrt(A C): within a rounding of singular (det ~ 0), power is ~0 along a line through
    the centre and those pairs are knives; at B = 0.9 sqrt(A C) power is clear of 0 off the centre and nothing is a
    knife.  The exact centre (power = 0 on both sides) is never one."""
    sc = _pixel_scene([0.5], sigma=1.0)
    st = h.oracle_forward(sc)
    co = st.conic_opacity.copy()
    co[0, 1] = np.sqrt(np.float64(co[0, 0]) * co[0, 2]) * b_scale
    st.conic_opacity[:] = co
    ke = A.knife_edges(st)
    assert (ke["pairs"] >= 1 and ke["splats"][0]) == knife
    assert not ke["pixels"][7, 7]
