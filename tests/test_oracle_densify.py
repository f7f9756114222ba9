"""CPU: oracle/densify.py (the gather-plan restatement the CUDA op follows) against the REAL reference densification
run on CPU: two random models (tests/golden/make_golden_densify.py -> densify_vectors.npz) and small models built on
its decision edges (make_golden_densify_edges.py -> densify_edges_vectors.npz)."""
import os

import numpy as np
import pytest

from oracle import densify as od

GOLD = os.path.join(os.path.dirname(__file__), "golden", "densify_vectors.npz")
EDGES = os.path.join(os.path.dirname(__file__), "golden", "densify_edges_vectors.npz")
EDGE_CASES = [str(c) for c in np.load(EDGES)["cases"]]


def load_case(case, path=GOLD):
    z = np.load(path)
    params = {n: z[f"{case}_in_{n}"] for n in od.NAMES}
    state = {n: (z[f"{case}_in_{n}_exp_avg"], z[f"{case}_in_{n}_exp_avg_sq"]) for n in od.NAMES}
    stats = {k: z[f"{case}_in_{k}"] for k in ("xyz_gradient_accum", "denom", "max_radii2D")}
    bound = f"{case}_in_binding" in z.files
    extra = dict(binding=z[f"{case}_in_binding"].astype(np.int64), binding_counter=z[f"{case}_in_binding_counter"],
                 face_scaling=z[f"{case}_in_face_scaling"]) if bound else {}
    want = {n: z[f"{case}_out_{n}"] for n in od.NAMES}
    want_state = {n: (z[f"{case}_out_{n}_exp_avg"], z[f"{case}_out_{n}_exp_avg_sq"]) for n in od.NAMES}
    want_b = (z[f"{case}_out_binding"], z[f"{case}_out_binding_counter"]) if bound else (None, None)
    return params, state, stats, z[f"{case}_hyper"], z[f"{case}_noise"], extra, want, want_state, want_b, z


@pytest.mark.parametrize("case", ["bound", "plain"])
def test_gather_plan_reproduces_the_reference_densification(case):
    params, state, stats, hyper, noise, extra, want, want_state, want_b, z = load_case(case)
    out_p, out_s, b, c, P2 = od.densify_and_prune(params, state, stats, hyper, noise, **extra)
    assert P2 == want["xyz"].shape[0]
    pl = od.plan(params, stats, hyper, **extra)
    assert pl["clone"].sum() > 0 and pl["split"].sum() > 0 and (~pl["keep_orig"] & ~pl["split"]).sum() > 0, \
        "fixture must exercise clone, split and prune"
    for n in od.NAMES:
        if n in ("xyz", "scaling"):   # children: a bmm / exp-log chain evaluated in a different association
            # (3-term dot products with cancellation: the error scales with the terms, i.e. with the largest entry)
            assert np.allclose(out_p[n], want[n], rtol=2e-6, atol=1e-6 * float(np.abs(want[n]).max())), n
        else:
            assert np.array_equal(out_p[n], want[n]), n
        assert np.array_equal(out_s[n][0], want_state[n][0]) and np.array_equal(out_s[n][1], want_state[n][1]), n
    if want_b[0] is not None:
        assert np.array_equal(b, want_b[0]) and np.array_equal(c, want_b[1])
        assert (c > 0).all() or (z[f"{case}_in_binding_counter"] == 0).any()
    # the statistics come back zeroed at the new length (densification_postfix)
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert z[f"{case}_out_{k}"].shape[0] == P2 and not z[f"{case}_out_{k}"].any()


def check_edge_rows(got_p, got_s, got_b, got_c, n_fixed, want, want_state, want_b):
    """Rows [0, n_fixed) (kept originals and clones) of every array, every row of the arrays a split child copies,
    both Adam moments, binding and binding_counter: bit for bit, NaN where the reference has NaN.  The children's
    xyz and scaling: the tolerance of the random fixtures, over the finite entries, with inf and NaN in place."""
    for n in od.NAMES:
        got, exp = got_p[n], want[n]
        assert got.shape == exp.shape, n
        if n in ("xyz", "scaling"):
            assert np.array_equal(got[:n_fixed], exp[:n_fixed], equal_nan=True), n
            fin = np.abs(exp[np.isfinite(exp)])
            atol = 1e-6 * float(fin.max()) if fin.size else 0.0
            assert np.allclose(got[n_fixed:], exp[n_fixed:], rtol=2e-6, atol=atol, equal_nan=True), n
        else:
            assert np.array_equal(got, exp, equal_nan=True), n
        assert np.array_equal(got_s[n][0], want_state[n][0], equal_nan=True), n + " exp_avg"
        assert np.array_equal(got_s[n][1], want_state[n][1], equal_nan=True), n + " exp_avg_sq"
    if want_b[0] is not None:
        assert np.array_equal(got_b, want_b[0]) and np.array_equal(got_c, want_b[1])


@pytest.mark.parametrize("case", EDGE_CASES)
def test_gather_plan_reproduces_the_reference_at_its_decision_edges(case):
    """Thresholds rounded as the reference rounds them, NaN and inf inputs, the face rule's boundaries, empty models."""
    params, state, stats, hyper, noise, extra, want, want_state, want_b, z = load_case(case, EDGES)
    assert hyper.dtype == np.float64
    pl = od.plan(params, stats, hyper, **extra)
    assert 2 * int(pl["split"].sum()) == noise.shape[0]
    out_p, out_s, b, c, P2 = od.densify_and_prune(params, state, stats, hyper, noise, **extra)
    assert P2 == want["xyz"].shape[0]
    n_fixed = int(pl["keep_orig"].sum() + pl["keep_clone"].sum())
    check_edge_rows(out_p, out_s, b, c, n_fixed, want, want_state, want_b)
