"""CPU: the oracle's per-splat preprocess and preprocess backward against the float64 projection of oracle/dense64.py
(`project`), splat by splat, on the edge scenes of tests/preprocess_scenes.py.

* The scenes reach every regime of the preprocess (a self-check, like test_corpus_reaches_every_path), and the float32
  restatement that decides the regimes reproduces the oracle's radii and conics bit for bit.
* Forward: the oracle's pixel centre, depth, conic and colour against project(), each within a few float32 roundings
  of the float64 value (the KNIFE_COND splats within kappa 2^-24 of their conic's size).
* Backward: the oracle's stage 5 and the float64 VJP driven by the same arbitrary per-splat upstream (random, one field
  at a time, zero): every splat row of every gradient within FLOOR of its own float64 magnitude (plus 4 kappa 2^-24
  for the KNIFE_COND splats).  That is the oracle's side of the per-splat gate the GPU test holds the kernels to
  (preprocess_scenes.gate_ratio).
* Mutations: wrong variants of the float64 chain (dense64.VARIANTS) are each rejected by the per-splat gate, which
  names the splats and their families; the tensor-wide gate of helpers.assert_grad_explained is run on the same
  gradients and its verdict printed beside it (run with -s).
"""
import numpy as np
import pytest

from oracle import dense64
from oracle import rasterizer as orc
from tests import helpers as h
from tests import preprocess_scenes as PS

ROUTES = [("shs", 3, 3, 0.7), ("shs", 2, 3, 1.0), ("shs", 1, 3, 1.3), ("shs", 0, 1, 1.0), ("colors_precomp", 0, 0, 1.0),
          ("cov3D_precomp", 3, 3, 1.0)]
_CACHE = {}


def _rid(r):
    return f"{r[0]}-deg{r[1]}of{r[2]}-mod{r[3]}"


def _case(route):
    if route not in _CACHE:
        name, deg, max_deg, mod = route
        sc = PS.edge_scene(route=name, sh_degree=deg, max_sh_degree=max_deg, scale_modifier=mod)
        cam = sc["cam"]
        st = orc.forward(sc["means3D"].numpy(), sc["opacities"].numpy(), cam.world_view_transform.numpy(),
                         cam.full_proj_transform.numpy(), cam.camera_center.numpy(), sc["W"], sc["H"], cam.tanfovx,
                         cam.tanfovy, sc["bg"].numpy(), **PS.oracle_kwargs(sc))
        pr = PS.f32_project(sc["means3D"].numpy(), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
                            sc["W"], sc["H"], cam.tanfovx, cam.tanfovy, st.cov3D)
        _CACHE[route] = (sc, st, pr)
    return _CACHE[route]


@pytest.mark.parametrize("route", [ROUTES[0], ROUTES[4], ROUTES[5]], ids=_rid)
def test_scenes_reach_every_regime(route):
    sc, st, pr = _case(route)
    kept = st.radii > 0
    # the float32 restatement the regimes are read from is the oracle's own arithmetic
    assert (pr["radius"][kept] == st.radii[kept]).all()
    a, b, c = pr["cov2d"].T
    inv = np.float32(1) / pr["det"][kept]
    assert (c[kept] * inv == st.conic_opacity[kept, 0]).all() and (-b[kept] * inv == st.conic_opacity[kept, 1]).all()
    reached = PS.regimes(sc, st)
    for name, m in reached.items():
        print(f"[regime] {_rid(route):<28s} {name:<46s} {int(m.sum())}")
    missing = [name for name, m in reached.items() if not m.any()]
    assert not missing, f"regimes no splat reaches: {missing}"
    assert set(sc["family"]) == {"guard", "near", "needle", "radius_edge", "offscreen", "scale", "quat", "colour", "plain"}


@pytest.mark.parametrize("route", ROUTES, ids=_rid)
def test_oracle_record_matches_float64_projection(route):
    import torch

    sc, st, pr32 = _case(route)
    keep = st.radii > 0
    inputs = {k: sc[k].double() for k in ("means3D", "scales", "rotations", "shs", "colors_precomp", "cov3D_precomp")
              if k in sc}
    if "colors_precomp" in sc:
        inputs.pop("shs")
    if "cov3D_precomp" in sc:
        inputs.pop("scales"), inputs.pop("rotations")
    pr = dense64.project(inputs.pop("means3D"), *PS.cam_args(sc), sh_degree=sc["sh_degree"],
                         scale_modifier=sc["scale_modifier"], guard_clamped=torch.from_numpy(pr32["guard"]),
                         colour_clamped=torch.from_numpy(st.clamped != 0), **inputs)
    fam = sc["family"]
    ill = PS.ill_kappa_of(st, pr32)
    W, H = sc["W"], sc["H"]

    def check(what, ora, ref, allow):
        err = np.abs(np.asarray(ora, np.float64) - ref)
        bad = np.nonzero(keep & ~(err <= allow).all(1))[0]
        worst = float((err / allow)[keep].max()) if keep.any() else 0.0
        print(f"[forward] {_rid(route):<28s} {what:<8s} worst error / allowance {worst:.2e}")
        assert not bad.size, (f"{what}: {bad.size} splats off; splat {bad[0]} ({fam[bad[0]]}): oracle {ora[bad[0]]} "
                              f"float64 {ref[bad[0]]}")

    pix = pr["pix"].numpy()
    check("pixel", st.xy, pix, 2.0 ** -20 * (np.abs(pix) + np.array([[W, H]])))
    check("depth", st.depths[:, None], pr["depth"].numpy()[:, None], 2.0 ** -22 * np.abs(pr["depth"].numpy()[:, None]))
    con = pr["conic"].numpy()
    size = np.sqrt(np.abs(con[:, 0] * con[:, 2]))[:, None] + np.abs(con)
    # det = a c - b^2 cancels: the roundings of a, b and c reach the conic amplified by cond2 = (|a c| + b^2) / det
    a, b, c = pr32["cov2d"].astype(np.float64).T
    cond2 = ((np.abs(a * c) + b * b) / np.abs(pr32["det"].astype(np.float64)))[:, None]
    check("conic", st.conic_opacity[:, :3], con, (2.0 ** -16 + (8.0 * cond2 + ill[:, None]) * 2.0 ** -24) * size)
    mag = 1.0 + (np.abs(sc["shs"].numpy()).sum(1) if "colors_precomp" not in sc else 0.0)
    check("rgb", st.rgb, pr["rgb"].numpy(), 2.0 ** -20 * mag)


KINDS = ["random", "one-hot:ndc", "one-hot:conic", "one-hot:opacity", "one-hot:rgb", "one-hot:z", "zero"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("route", ROUTES, ids=_rid)
def test_oracle_backward_matches_float64_vjp(route, kind):
    sc, st, pr = _case(route)
    keep = st.radii > 0
    up = PS.upstream(len(keep), kind, seed=7, with_z=True)
    f64 = PS.vjp64(sc, up, keep, pr["guard"], st.clamped, pr["conic_dropped"])
    ora = PS.oracle_vjp(sc, st, up)
    ik = PS.ill_kappa_of(st, pr)
    for name, ref in f64.items():
        # the oracle against float64 alone: its error within FLOOR (+ kappa 2^-24) of each row's own size
        ratio = PS.assert_gate(name, ora[name], ref, ref, ik, sc["family"], f"{_rid(route)} {kind} oracle")
        p50, p99, worst = PS.percentiles(ratio)
        print(f"[oracle vs float64] {_rid(route):<28s} {kind:<16s} dL/d{name:<15s} p50 {p50:.2e} p99 {p99:.2e} "
              f"max {worst:.2e}")
        assert (np.asarray(ora[name]).reshape(len(keep), -1)[~keep] == 0).all(), f"{name}: culled splats not zero"
        if kind == "zero":
            assert (np.asarray(ora[name]) == 0).all()


@pytest.mark.parametrize("variant", dense64.VARIANTS)
def test_per_splat_gate_rejects_wrong_backwards(variant):
    """A wrong float64 chain in the place of the kernel: the per-splat gate rejects it; the tensor-wide gate's verdict
    on the same gradients is printed beside it."""
    sc, st, pr = _case(ROUTES[0])
    keep = st.radii > 0
    up = PS.upstream(len(keep), "random", seed=11, with_z=True)
    f64 = PS.vjp64(sc, up, keep, pr["guard"], st.clamped, pr["conic_dropped"])
    bad = PS.vjp64(sc, up, keep, pr["guard"], st.clamped, pr["conic_dropped"], variant=variant)
    ora = PS.oracle_vjp(sc, st, up)
    ik = PS.ill_kappa_of(st, pr)
    rejected = {}
    for name, ref in f64.items():
        dev = bad[name].astype(np.float32)
        ratio = PS.gate_ratio(dev, ora[name], ref, ik)
        n_rej = int((~(ratio <= 1.0)).sum())
        try:
            h.assert_grad_explained(dev, ref, ik > 0, f"{variant} dL/d{name}")
            tensor = "passes"
        except AssertionError:
            tensor = "rejects"
        if n_rej or tensor == "rejects":
            print(f"[mutation] {variant:<22s} dL/d{name:<12s} per-splat gate rejects {n_rej:>5d} splats "
                  f"(families {sorted(set(sc['family'][~(ratio <= 1.0)]))}); tensor gate {tensor}")
        rejected[name] = n_rej
    assert sum(rejected.values()) > 0, f"{variant}: the per-splat gate accepts the wrong backward"
