"""Generates tests/golden/densify_edges_vectors.npz: the REAL reference densification (GaussianModel.densify_and_prune,
scene/gaussian_model.py:334-519) run on CPU tensors on small models built to sit on its decision edges.  Same harness as
make_golden_densify.py (factory device keywords dropped, torch.normal fed recorded noise).

Every edge is placed where the float32 value is exact in any libm: raw scaling 0 (exp = 1, so the world scale IS the
face scaling), raw opacity 0 / +-100 (sigmoid = 1/2, 1, 0) and IEEE division for the gradient.  Split children keep
their world scale at least a factor of 2 away from 0.1 * extent.  Each case asserts that its edge decides something in
the reference run -- a fixture that cannot tell two arithmetics apart tests nothing.

Cases (name -> inputs, outputs, noise and float64 hyper-parameters, prefixed `<name>_`; the names are in `cases`):
  thr_gap_*    percent_dense * extent formed in double and rounded once (the reference: a float32 tensor compared with
               a Python product) vs the float product of the rounded factors; splats on both, on their neighbours, with
               the gradient exactly at max_grad, one ulp either side, 0/0, x/0 and -x/0
  ws_gap_*     0.1 * extent likewise, for the world-size prune (max_screen_size 20, None, 0); split parents whose
               children land well above / below it
  opacity_*    sigmoid(0) = 1/2 against min_opacity 1/2, the float32 above it and the float64 above it; +-100
  face_rule    every boundary of `counter + delta - candidates` in {0, 1} of the all-or-nothing face rule
  poisoned     NaN / inf in scales, opacity and accumulated gradient, a zero quaternion on a split parent
  degenerate_* P = 0 (bound and plain), every splat pruned, every splat split, no change; SH degrees 0, 1 and 3

    python tests/golden/make_golden_densify_edges.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from tests import ref_import  # noqa: E402
from tests.golden.make_golden_densify import ATTR, _Patches, build_model, snapshot  # noqa: E402

f32 = np.float32
PD = 0.01          # percent_dense of the reference's OptimizationParams
MAX_GRAD = 0.0002  # densify_grad_threshold
NAN, INF = float("nan"), float("inf")


def up(x):
    return f32(np.nextafter(f32(x), f32(np.inf)))


def down(x):
    return f32(np.nextafter(f32(x), f32(-np.inf)))


def thresholds(extent):
    """(reference, float product) for the clone/split threshold and the world-size threshold."""
    return (f32(PD * extent), f32(f32(PD) * f32(extent)), f32(0.1 * extent), f32(f32(0.1) * f32(extent)))


def pick_extents():
    """Deterministic extents of three decimals: the first two where each threshold's two roundings differ in each
    direction, and the first two where all four agree."""
    want = {k: [] for k in ("thr_lo", "thr_hi", "big_lo", "big_hi", "agree")}
    for ext in (round(0.5 + 0.001 * k, 3) for k in range(4500)):
        tr, tk, br, bk = thresholds(ext)
        for key, hit in (("thr_lo", tk < tr), ("thr_hi", tk > tr), ("big_lo", bk < br), ("big_hi", bk > br),
                         ("agree", tk == tr and bk == br)):
            if hit and len(want[key]) < 2:
                want[key].append(ext)
    assert all(len(v) == 2 for v in want.values()), want
    return want


def model(P, deg, seed, binding=None, face_scaling=None):
    """build_model's random splats, Adam moments and statistics; bound to `binding` when given (a consistent
    binding_counter, identity face frames: get_xyz is only asked for its row count)."""
    m = build_model(P, 0, deg, False, seed)
    if binding is not None:
        F = len(face_scaling)
        m.binding = torch.as_tensor(np.asarray(binding, np.int64))
        m.binding_counter = torch.bincount(m.binding, minlength=F).to(torch.int32)
        m.face_scaling = torch.tensor(np.asarray(face_scaling, f32)).reshape(F, 1)
        m.face_center = torch.zeros(F, 3)
        m.face_orien_mat = torch.eye(3).repeat(F, 1, 1)
        m.face_orien_quat = torch.tensor([1.0, 0.0, 0.0, 0.0]).repeat(F, 1)
    m.percent_dense = PD
    return m


@torch.no_grad()
def put(m, name, rows, value):
    """Writes raw parameter rows in place (the optimizer state is keyed by the Parameter object)."""
    getattr(m, ATTR[name])[rows] = torch.as_tensor(value, dtype=torch.float32)


def grads(m, accum, denom):
    m.xyz_gradient_accum = torch.tensor(np.asarray(accum, f32)).reshape(-1, 1)
    m.denom = torch.tensor(np.asarray(denom, f32)).reshape(-1, 1)


class Run:
    def __init__(self):
        self.out, self.cases = {}, []

    def __call__(self, name, m, min_opacity, extent, screen):
        """Runs the reference on `m` (in place); returns (P_out, per-face output rows, per-face output rows whose raw
        scaling is untouched, i.e. kept originals and clones) for the assertions."""
        snapshot(m, f"{name}_in", self.out)
        with _Patches(torch.Generator().manual_seed(1000 + len(self.cases))) as pt:
            m.densify_and_prune(MAX_GRAD, min_opacity, extent, screen)
        snapshot(m, f"{name}_out", self.out)
        self.out[f"{name}_noise"] = (torch.cat(pt.noise) if pt.noise else torch.zeros(0, 3)).numpy()
        self.out[f"{name}_hyper"] = np.array([MAX_GRAD, min_opacity, extent, -1.0 if screen is None else float(screen),
                                              m.percent_dense], np.float64)
        self.cases.append(name)
        P_out = m._xyz.shape[0]
        print(f"{name:16s} P {self.out[f'{name}_in_xyz'].shape[0]:3d} -> {P_out:3d}, split parents "
              f"{self.out[f'{name}_noise'].shape[0] // 2}")
        if getattr(m, "binding", None) is None:
            return P_out, None, None
        F = m.binding_counter.shape[0]
        b = m.binding.numpy()
        scale_in = {r.tobytes() for r in self.out[f"{name}_in_scaling"]}      # bytes: NaN rows match themselves
        untouched = np.array([r.tobytes() in scale_in for r in m._scaling.detach().numpy()], bool)
        return P_out, np.bincount(b, minlength=F), np.bincount(b[untouched], minlength=F)


def thr_gap(run, ext, tag):
    """One splat per face, raw scaling 0: world scale = face scaling exactly.  Face scalings: the reference threshold,
    its two float neighbours and the float-product threshold; gradients: exactly max_grad, one ulp either side, 0/0
    (NaN -> 0), x/0 (inf) and -x/0 (-inf: clones by |g|, never splits)."""
    tr, tk, _, _ = thresholds(ext)
    g = f32(MAX_GRAD)
    sizes = [tr, down(tr), up(tr), tk]
    grad = [(g, 1.0), (down(g), 1.0), (up(g), 1.0), (0.0, 0.0), (g, 0.0), (-g, 0.0)]
    rows = [(s, a, d) for s in sizes for a, d in grad]
    P = len(rows)
    m = model(P, 1, 20 + len(run.cases), binding=np.arange(P), face_scaling=[r[0] for r in rows])
    put(m, "scaling", slice(None), 0.0)
    put(m, "opacity", slice(None), 5.0)
    grads(m, [r[1] for r in rows], [r[2] for r in rows])
    _, rows_out, untouched = run(f"thr_gap_{tag}", m, 0.005, ext, None)
    # per face: clone = original + clone (2 untouched rows), split = two children (2 rows, none untouched)
    cloned, split = untouched == 2, (rows_out == 2) & (untouched == 0)
    fs = np.array([r[0] for r in rows], f32)
    g_in = np.array([f32(r[1]) / f32(r[2]) if r[2] else (np.sign(r[1]) * np.inf if r[1] else 0.0) for r in rows], f32)
    for thr, what in ((tr, "reference"), (tk, "float product")):
        want_clone, want_split = (np.abs(g_in) >= g) & (fs <= thr), (g_in >= g) & (fs > thr)
        if what == "reference":
            assert (cloned == want_clone).all() and (split == want_split).all(), "reference threshold mispredicted"
        elif tk != tr:
            assert (cloned != want_clone).any() and (split != want_split).any(), "float product decides the same"
    assert cloned.any() and split.any() and (~cloned & ~split).any()


def ws_gap(run, ext, screen, tag):
    """Two splats per face: an edge splat and a healthy one (so the face rule lets the edge splat go).  Edge splats
    with zero gradient at the reference world-size threshold, its neighbours and the float product; split parents
    whose children (world scale / 1.6) land 3x above and 3.2x below 0.1 * extent."""
    _, _, br, bk = thresholds(ext)
    edge = [(br, 0.0), (down(br), 0.0), (up(br), 0.0), (bk, 0.0), (f32(0.5 * ext), 1.0), (f32(0.05 * ext), 1.0)]
    F = len(edge)
    binding = np.repeat(np.arange(F), 2)
    m = model(2 * F, 1, 40 + len(run.cases), binding=binding, face_scaling=[e[0] for e in edge])
    put(m, "scaling", slice(0, None, 2), 0.0)
    put(m, "scaling", slice(1, None, 2), -3.0)                  # healthy: world scale ~0.05 x the edge's
    put(m, "opacity", slice(None), 5.0)
    grads(m, np.stack([[f32(MAX_GRAD) * e[1] for e in edge], np.zeros(F)], 1).reshape(-1), np.ones(2 * F))
    _, rows_out, _ = run(f"ws_gap_{tag}", m, 0.005, ext, screen)
    edge_kept = rows_out - 1                                    # the healthy splat always stays
    fs = np.array([e[0] for e in edge], f32)
    on = bool(screen)
    assert (edge_kept[:4] == np.where(on & (fs[:4] > br), 0, 1)).all(), "reference world-size threshold mispredicted"
    assert (edge_kept[4:] == ([0, 2] if on else [2, 2])).all(), "children above 0.1 extent must go, below must stay"
    if on and bk != br:
        assert (edge_kept[:4] != np.where(fs[:4] > bk, 0, 1)).any(), "float product decides the same"


def opacity(run, min_opacity, tag):
    """Plain model: raw opacity 0 (sigmoid = 1/2), +100 (1), -100 (0); clone and split parents with raw opacity 0."""
    m = model(8, 0, 60 + len(run.cases))
    put(m, "opacity", slice(None), torch.tensor([0.0, 0.0, 100.0, -100.0, 0.0, 0.0, 100.0, 3.0]).reshape(8, 1))
    put(m, "scaling", slice(None), -1.5)                       # world 0.22 > 0.01 extent: split when the gradient is high
    put(m, "scaling", [4, 6], -7.0)                            # world 9e-4: clone
    grads(m, [0, 0, 0, 0, 1, 1, 1, 0], np.ones(8))
    P_out, _, _ = run(f"opacity_{tag}", m, min_opacity, 1.0, None)
    half_pruned = f32(min_opacity) > f32(0.5)
    # rows 0, 1, clone parent 4 and its clone, children of 5: kept unless 1/2 < min_opacity; 2, 6 and its clone, 7
    assert P_out == (0 if half_pruned else 6) + 4, P_out


def face_rule(run):
    """Faces (raw scaling 0, so fs alone sets the size; low = raw opacity -10, healthy = +5 with zero gradient):
      0  a lone low-opacity clone parent         counter 1 + delta 1 - candidates 2 = 0 -> both stay
      1  a lone low-opacity split parent         1 + 1 - 2 = 0 -> both children stay
      2  two low + one healthy                   3 + 0 - 2 = 1 -> both low go
      3  two low                                 2 + 0 - 2 = 0 -> both stay
      4  a low clone parent + one healthy        2 + 1 - 2 = 1 -> parent and clone go
      5  a low split parent + one healthy        2 + 1 - 2 = 1 -> both children go
      6  a low clone and a low split parent      2 + 2 - 4 = 0 -> all four stay
      7  no splats (counter 0)
      8  a healthy clone parent + a low splat    2 + 1 - 1 = 2 -> the low splat goes"""
    thr = f32(PD * 1.0)
    small, large = f32(0.25) * thr, f32(4.0) * thr             # clone / split sizes; 0.04 < 0.1 extent / 2
    spec = [  # (face, face scaling, raw opacity, gradient)
        (0, small, -10, 1), (1, large, -10, 1), (2, small, -10, 0), (2, small, -10, 0), (2, small, 5, 0),
        (3, large, -10, 0), (3, large, -10, 0), (4, small, -10, 1), (4, small, 5, 0), (5, large, -10, 1),
        (5, large, 5, 0), (6, small, -10, 1), (8, small, 5, 1), (8, small, -10, 0)]
    fs = np.full(9, small, f32)
    for f, s, _, _ in spec:
        fs[f] = s
    fs[6] = small
    binding = np.array([s[0] for s in spec] + [6])
    P = len(binding)
    m = model(P, 1, 80, binding=binding, face_scaling=fs)
    put(m, "scaling", slice(None), 0.0)
    put(m, "scaling", P - 1, torch.tensor([2.8, 0.0, 0.0]))   # face 6's split parent: world 16.4 fs = 0.041 > thr
    put(m, "opacity", slice(None), torch.tensor([float(s[2]) for s in spec] + [-10.0]).reshape(P, 1))
    grads(m, [float(s[3]) for s in spec] + [1.0], np.ones(P))
    _, rows_out, _ = run("face_rule", m, 0.005, 1.0, 20)
    assert rows_out.tolist() == [2, 2, 1, 2, 1, 1, 4, 0, 2], rows_out.tolist()


def poisoned(run):
    """One poisoned splat per face, each with a healthy companion (raw scaling -3, zero gradient) unless noted.
      0  scale (0, NaN, 0), fs < thr, gradient high     max is NaN: no clone (fmaxf would clone)
      1  scale (0, NaN, 0), thr < fs < 0.1 extent       no split
      2  scale (0, NaN, 0), fs > 0.1 extent, no gradient  no world-size prune
      3  scale (NaN, NaN, NaN), gradient high           nothing (a maximum seeded below zero would clone)
      4  NaN opacity, gradient high, small: cloned, never pruned by opacity
      5  NaN accumulated gradient, large: nothing
      6  inf accumulated gradient (denom 1), large: split
      7  raw scaling (100, 0, 0), lone on its face: exp = inf, split; children at inf scale (kept by the face rule)
      8  zero quaternion, split: the children's positions are NaN"""
    thr, big = f32(PD), f32(0.1)
    fs = np.array([thr / 4, thr * 4, big * 2, thr * 4, thr / 4, thr * 4, thr * 4, thr, thr * 4], f32)
    F = len(fs)
    lone = {7}
    binding = np.concatenate([np.arange(F), [f for f in range(F) if f not in lone]])
    P = len(binding)
    m = model(P, 1, 90, binding=binding, face_scaling=fs)
    put(m, "scaling", slice(0, F), 0.0)
    put(m, "scaling", slice(F, None), -3.0)
    put(m, "opacity", slice(None), 5.0)
    put(m, "scaling", [0, 1, 2], torch.tensor([0.0, NAN, 0.0]))
    put(m, "scaling", 3, NAN)
    put(m, "opacity", 4, NAN)
    put(m, "scaling", 7, torch.tensor([100.0, 0.0, 0.0]))
    put(m, "rotation", 8, 0.0)
    accum = np.zeros(P, f32)
    accum[[0, 1, 3, 4, 7, 8]] = 1.0
    accum[5], accum[6] = NAN, INF
    grads(m, accum, np.ones(P))
    _, rows_out, untouched = run("poisoned", m, 0.005, 1.0, 20)
    assert rows_out.tolist() == [2, 2, 2, 2, 3, 2, 3, 2, 3], rows_out.tolist()
    assert untouched.tolist() == [2, 2, 2, 2, 3, 2, 1, 0, 1], untouched.tolist()
    xyz = m._xyz.detach().numpy()
    assert np.isnan(xyz).any(axis=1).sum() == 2 and np.isinf(m._scaling.detach().numpy()).any(axis=1).sum() == 2


def degenerate(run):
    m = model(0, 1, 100, binding=np.zeros(0, np.int64), face_scaling=np.full(5, 0.01, f32))
    assert run("degenerate_empty_bound", m, 0.005, 1.0, 20)[1].tolist() == [0] * 5
    assert run("degenerate_empty_plain", model(0, 0, 101), 0.005, 1.0, None)[0] == 0
    m = model(12, 1, 102)
    put(m, "opacity", slice(None), -10.0)
    grads(m, np.r_[np.ones(6), np.zeros(6)], np.ones(12))       # clones and children are pruned with their parents
    put(m, "scaling", slice(0, 3), -7.0)
    assert run("degenerate_all_pruned", m, 0.005, 1.0, 20)[0] == 0
    m = model(10, 3, 103)
    put(m, "scaling", slice(None), -1.5)
    put(m, "opacity", slice(None), 5.0)
    grads(m, np.ones(10), np.ones(10))
    assert run("degenerate_all_split", m, 0.005, 1.0, None)[0] == 20
    m = model(10, 0, 104)
    put(m, "opacity", slice(None), 5.0)
    grads(m, np.zeros(10), np.r_[np.ones(5), np.zeros(5)])
    assert run("degenerate_unchanged", m, 0.005, 1.0, None)[0] == 10
    m = model(16, 0, 105)                                      # SH degree 0: no _features_rest columns
    put(m, "opacity", slice(None), 5.0)
    put(m, "scaling", slice(0, 8), -7.0)
    put(m, "scaling", slice(8, None), -1.5)
    grads(m, np.r_[np.ones(4), np.zeros(4), np.ones(4), np.zeros(4)], np.ones(16))
    assert run("degenerate_sh0_mixed", m, 0.005, 1.0, None)[0] == 16 + 4 + 4


def main():
    ref_import.prepare()
    run = Run()
    ext = pick_extents()
    print("extents", ext)
    for tag, e in (("lo", ext["thr_lo"][0]), ("lo2", ext["thr_lo"][1]), ("hi", ext["thr_hi"][0]),
                   ("agree", ext["agree"][0])):
        thr_gap(run, e, tag)
    for screen, tag in ((20, "lo"), (None, "lo_none"), (0, "lo_zero")):
        ws_gap(run, ext["big_lo"][0], screen, tag)
    ws_gap(run, ext["big_hi"][0], 20, "hi")
    ws_gap(run, ext["agree"][1], 20, "agree")
    for v, tag in ((0.5, "half"), (float(up(0.5)), "f32_above"), (float(np.nextafter(0.5, 1.0)), "f64_above")):
        opacity(run, v, tag)
    face_rule(run)
    poisoned(run)
    degenerate(run)
    run.out["cases"] = np.array(run.cases)
    path = os.path.join(HERE, "densify_edges_vectors.npz")
    np.savez_compressed(path, **run.out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
