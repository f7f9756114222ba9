"""CPU: the composed training step of tests/train_step_oracle.py, before any GPU is involved.

  * the float64 step equals central finite differences of its own loss, along random directions of every raw splat
    parameter and every posed FLAME parameter, with both regulariser settings: the yardstick differentiates what it
    computes;
  * condition A: the float32 reference-order step passes every gate against the float64 step -- no gate is stricter
    than the reference itself;
  * condition B: each deliberately wrong variant of the float64 step (train_step_oracle.MUTATIONS) fails a gate on the
    same scene -- the gates can see the bug each stands for;
  * the scene reaches the regimes tests/test_gpu_train_step.py exists for, asserted on the oracles' own state."""
import functools

import numpy as np
import pytest
import torch

from tests import flame_oracle as fo
from tests import helpers as h
from tests import train_step_oracle as T

# the scenes of tests/test_gpu_train_step.py: (timestep, active SH degree, metric regularisers)
SCENES = [(2, 3, False), (4, 1, True), (6, 3, True)]


@functools.lru_cache(maxsize=None)
def _scene():
    return T.scene()


def _flags(sc, sh, metric):
    return T.metric_flags(sc, sh) if metric else T.flags(sh)


@functools.lru_cache(maxsize=None)
def _pair(t, sh, metric):
    sc = _scene()
    return T.run_pair(sc, t, _flags(sc, sh, metric))


# ---- the float64 step against finite differences ------------------------------------------------------------------
def _decisions(r):
    """Every discrete decision of a float64 step: blend acceptance and stops, the clamps, the regulariser hinges and
    the sign of each L1 term."""
    a = r["aux"]
    return [a["keep"], a["alpha_clamped"], a["colour_clamped"], a["guard_clamped"],
            torch.from_numpy(r["reg_active"][0]), torch.from_numpy(r["reg_active"][1]), torch.from_numpy(r["l1_sign"])]


@pytest.mark.parametrize("metric", [False, True], ids=["default-regularisers", "metric-regularisers"])
def test_float64_step_equals_central_differences(metric):
    sc = T.scene(P=100, W=24, H=16, seed=1, scale_shift=2.0, hot=(), far=0.0)
    # the render passes the gradient straight through min(0.99, alpha) and the guard band's clamp, as the reference
    # does (oracle/dense64.py): the derivative is only the loss's own where neither is reached
    sc["params"]["_opacity"].clamp_(max=4.0)
    t = 2
    fl = _flags(sc, 3, metric)
    p64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sc["params"].items()}
    f64 = {k: v.double() for k, v in sc["flame_param"].items()}
    args = (sc["assets"], sc["cam"], sc["gt"], fl, torch.float64)
    pin = T.step(sc["params"], sc["flame_param"], t, *args[:4], torch.float32)["pin"]
    base = T.step(p64, f64, t, *args, pin=pin)
    assert (base["radii"] > 0).sum() >= 50 and base["parts"]["xyz"] > 0 and base["parts"]["scale"] > 0
    d0 = _decisions(base)
    assert not (base["aux"]["alpha_clamped"] & base["aux"]["keep"]).any() and not base["aux"]["guard_clamped"].any()
    gen = torch.Generator().manual_seed(11)
    groups = [("raw", k) for k in T.RAW] + [("flame", k) for k in fo.POSED]
    eps = 1e-6
    for kind, k in groups:
        src = p64 if kind == "raw" else f64
        for _ in range(2):
            d = torch.zeros_like(src[k])
            if kind == "raw":
                d = torch.randn(src[k].shape, generator=gen, dtype=torch.float64)
            else:
                d[t] = torch.randn(src[k].shape[1:], generator=gen, dtype=torch.float64)
            d = d / d.norm()
            ad = float((torch.from_numpy(base["grads"][k] if kind == "raw" else base["flame"][k]) * d).sum())
            loss = []
            for sgn in (1, -1):
                moved = dict(src)
                moved[k] = src[k] + sgn * eps * d
                r = T.step(moved, f64, t, *args, pin=pin) if kind == "raw" else T.step(p64, moved, t, *args, pin=pin)
                for x, y in zip(_decisions(r), d0):
                    assert torch.equal(x, y), f"d/d{k}: the step of {eps} crosses a threshold"
                loss.append(r["parts"]["total"])
            fd = (loss[0] - loss[1]) / (2 * eps)
            print(f"[fd] {k:<16s} autograd {ad:+.9e} central difference {fd:+.9e}")
            assert abs(fd - ad) <= 1e-6 * abs(ad) + 1e-9, f"d/d{k}: autograd {ad:.9e}, finite difference {fd:.9e}"


# ---- the gates: condition A and condition B ---------------------------------------------------------------------
@pytest.mark.parametrize("t,sh,metric", SCENES)
def test_float32_reference_passes_every_gate(t, sh, metric):
    r32, r64 = _pair(t, sh, metric)
    recs = T.gates(r32, r64, t)
    T.report(f"fp32 reference t={t} sh={sh} metric={metric}", recs)
    assert not T.failed(recs), f"the float32 reference fails {T.failed(recs)}: a gate is stricter than the reference"


@pytest.mark.parametrize("mutation", sorted(T.MUTATIONS))
def test_each_mutation_fails_a_gate(mutation):
    t, sh, metric = SCENES[1]   # the metric scene: every mutation applies to it
    sc = _scene()
    r32, r64 = _pair(t, sh, metric)
    rm = T.step(sc["params"], sc["flame_param"], t, sc["assets"], sc["cam"], sc["gt"], _flags(sc, sh, metric),
                torch.float64, pin=r32["pin"], mutation=mutation)
    bad = T.failed(T.gates(rm, r64, t))
    print(f"[mutation] ({mutation}) {T.MUTATIONS[mutation]}: rejected by {bad}")
    assert bad, f"mutation ({mutation}) {T.MUTATIONS[mutation]} passes every gate"
    expect = {"a": "dL/d_xyz", "b": "dL/dverts", "c": "dL/d_scaling", "d": "dL/dverts", "e": "dL/dmeans2D",
              "f": "dL/dverts"}[mutation]
    assert expect in bad, f"mutation ({mutation}) is not caught by the {expect} gate"


# ---- regimes ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [False, True], ids=["default-regularisers", "metric-regularisers"])
def test_scene_reaches_its_regimes(metric):
    sc = _scene()
    t, sh = (2, 3) if not metric else (4, 1)
    r32, r64 = _pair(t, sh, metric)
    g = T.regimes(sc["params"], sc["assets"]["faces"].shape[0], r64, r32)
    print(f"[regimes] metric={metric} {g}")
    assert g["max_chunks"] >= 4, "no face spans four chunks of the per-face reduction (more than 48 splats)"
    assert g["empty_face_frac"] > 0.5, "most faces must own no splat"
    assert g["mean_contrib"] >= 3
    assert g["low_T_frac"] >= 0.1
    assert g["xyz_active"] >= 0.05 and g["scale_active"] >= 0.05, "a regulariser term is zero on most splats"
    assert g["radius0"] > 0 and g["faint"] > 0
    # the pinned float64 render and the float32 oracle agree on the image: the pin holds the same splats in place
    # (a few pixels take an alpha >= 1/255 or T < 1e-4 decision the other way: knife edges of float32 against float64)
    h.assert_image_close(r32["image"], r64["image"], "float32 oracle vs pinned float64 render", frac=5e-4)
    assert np.array_equal(r64["radii"], r32["radii"])
