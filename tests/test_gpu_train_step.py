"""-m gpu: the whole mesh-bound training step on the device against the float64 step of tests/train_step_oracle.py.

The chain the float64 step pins end to end: photometric loss and the two binding regularisers -> dL/dimage -> blend
backward -> fused bound preprocess backward (raw splat gradients and the per-face dL/d{face_center, face_orien_mat,
face_scaling}, summed per face) -> face_frame backward -> dL/dverts -> FLAME backward -> dL/d{expr, rotation, neck,
jaw, eyes, translation}, and the viewspace gradient that feeds the densification statistics.  Three routes: the eager
step, one GraphedFrame replay of it, and the eager step with the per-face gradients summed by per-splat atomics
instead of the CSR chunk reduction.  The gates are train_step_oracle's, proven on the CPU by
tests/test_oracle_train_step.py (the float32 reference passes them, each mutation fails them); the float32
reference's tolerance ratios are printed next to the CUDA ones."""
import functools

import numpy as np
import pytest
import torch

from tests import flame_oracle as fo
from tests import train_step_oracle as T

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ATTR = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
# (timestep, active SH degree, metric regularisers): a generic posed row, the exactly-zero-pose row and the 2.5 rad
# row; SH degree 3, and 1 over 16 stored coefficients; the regularisers at their defaults and metric
SCENES = [(2, 3, False), (4, 1, True), (6, 3, True), (4, 3, False), (2, 1, True)]


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


@functools.lru_cache(maxsize=None)
def _scene():
    return T.scene()


def _flags(sc, sh, metric):
    return T.metric_flags(sc, sh) if metric else T.flags(sh)


def _lbs(a):
    import gaussianavatars_b200 as g
    return g.FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                                  a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=DEV)


def _model(sc, sh):
    from gaussianavatars_b200.model import MeshBoundGaussians
    p = {k: v.to(DEV).clone().contiguous() for k, v in sc["flame_param"].items()}
    for k in fo.POSED:
        p[k].requires_grad_(True)
    pc = MeshBoundGaussians(sc["params"], 3, None, None, device=DEV, requires_grad=True, flame=_lbs(sc["assets"]),
                            flame_param=p)
    for attr in ATTR:
        setattr(pc, attr, torch.nn.Parameter(getattr(pc, attr).detach().clone()))
    pc.active_sh_degree = sh
    return pc


def _n(x):
    return x.detach().double().cpu().numpy()


def _eager(sc, t, fl):
    """The eager step on the device; also the float32 activation the fused forward computed (bind_activate)."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.renderer import render
    pc = _model(sc, fl["sh_degree"])
    pc.select_mesh_by_timestep(t)
    pc.verts.retain_grad()
    out = render(sc["cam"].to(DEV), pc, Pipe, torch.tensor(fl["bg"], device=DEV))
    photo, parts = g.photometric_loss(out["render"], sc["gt"].to(DEV), fl["lambda_dssim"], return_parts=True)
    lx, ls = g.binding_regularizers(pc._xyz, pc._scaling, out["radii"], pc.binding, pc.face_scaling, **T.reg_kwargs(fl))
    total = photo + lx + ls
    total.backward()
    torch.cuda.synchronize()
    with torch.no_grad():
        act = g.bind_activate(1.0, pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc.binding, pc.face_center,
                              pc.face_orien_mat, pc.face_scaling)
    parts = parts.double().cpu()
    res = dict(parts=dict(l1=float(parts[0]), ssim=float(parts[1]), xyz=float(lx.detach()), scale=float(ls.detach()),
                         total=float(total.detach())),
               grads={**{k: _n(getattr(pc, k).grad) for k in ATTR}, "means2D": _n(out["viewspace_points"].grad),
                      "verts": _n(pc.verts.grad)},
               flame={k: _n(pc.flame_param[k].grad) for k in fo.POSED}, radii=out["radii"].cpu().numpy(),
               image=_n(out["render"]))
    shs = torch.cat((pc._features_dc, pc._features_rest), dim=1).detach()
    return res, act, shs


def _graphed(sc, t, fl):
    """One GraphedFrame replay of the same step, from zeroed densification statistics and without an optimiser."""
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    pc = _model(sc, fl["sh_degree"])
    P = pc._xyz.shape[0]
    pc.xyz_gradient_accum = torch.zeros((P, 1), device=DEV)
    pc.denom = torch.zeros((P, 1), device=DEV)
    pc.max_radii2D = torch.zeros((P,), device=DEV)
    cam = sc["cam"]
    fr = GraphedFrame(pc, sc["W"], sc["H"], cam.FoVx, cam.FoVy, torch.tensor(fl["bg"]), loss="photometric",
                      lambda_dssim=fl["lambda_dssim"], regularizers=T.reg_kwargs(fl), densify_stats=True)
    fr.set_inputs(camera=camera_block(cam).to(DEV), gt_u8=sc["gt"].to(DEV), timestep=t)
    fr.run()
    torch.cuda.synchronize()
    assert not fr.overflowed() and fr.replays == 1
    return dict(parts=dict(total=float(fr.loss)),
                grads={**{k: _n(getattr(pc, k).grad) for k in ATTR}, "means2D": _n(fr.viewspace_points.grad)},
                flame={k: _n(pc.flame_param[k].grad) for k in fo.POSED},
                xyz_gradient_accum=_n(pc.xyz_gradient_accum), denom=_n(pc.denom), max_radii2D=_n(pc.max_radii2D),
                radii=fr.radii.cpu().numpy())


def _references(sc, t, sh, metric, fl, act, shs):
    """The C oracle's forward on the CUDA-exported activation, the float64 step pinned to it, the float32 reference
    step and the float32 reference's gate records."""
    means3D, opac, scales, cov = act
    st = T.oracle_forward_on(means3D, opac, sc["cam"], sc["W"], sc["H"], fl, shs, cov3D=cov)
    args = (sc["params"], sc["flame_param"], t, sc["assets"], sc["cam"], sc["gt"], fl)
    r64 = T.step(*args, torch.float64, pin=T.pin_of(st))
    r32 = T.step(*args, torch.float32)
    return st, r64, r32, T.gates(r32, r64, t)


def _array(res, what, t):
    """The array a vertex or FLAME gate record `what` compares (row t of a FLAME gradient), or None."""
    if what == "dL/dverts":
        return res["grads"]["verts"]
    for k in fo.POSED:
        if what == f"dL/d{k}[t]":
            return res["flame"][k][t]
    return None


def _check(title, got, r64, r32, ref_recs, t):
    """Every gate of train_step_oracle; a vertex or FLAME gate the fixed tolerance rejects is passed only if the
    error stays within twice the float32 reference's on the same array (the rule of tests/test_gpu_flame.py: at
    2.5 rad per joint the reference's own float32 error reaches the fixed gate)."""
    recs = T.gates(got, r64, t)
    ref = {r["what"]: r for r in ref_recs}
    bad = []
    for r in recs:
        f32 = ref.get(r["what"])
        extra = f"   fp32 reference worst={f32['worst']:.2e}" if f32 else ""
        print(f"[train-step] {title:<40s} {r['what']:<20s} tol-ratio p50={r['p50']:.2e} p99.9={r['p999']:.2e} "
              f"worst={r['worst']:.2e} outliers={r['outliers']}/{r['allowed']}{extra}")
        if r["ok"]:
            continue
        a = _array(got, r["what"], t)
        if a is not None and "not zero" not in r["what"]:
            ref64 = _array(r64, r["what"], t)
            e_c = float(np.abs(np.asarray(a, np.float64) - ref64).max())
            e_32 = float(np.abs(np.asarray(_array(r32, r["what"], t), np.float64) - ref64).max())
            print(f"[train-step] {title:<40s} {r['what']:<20s} beyond the fixed gate: max|d| {e_c:.3e}, "
                  f"2 x fp32 reference {2 * e_32:.3e}")
            if e_c <= 2 * e_32:
                continue
        bad.append(r["what"])
    assert not bad, f"{title}: fails {bad}"


@pytest.mark.parametrize("t,sh,metric", SCENES)
def test_eager_and_graphed_steps_match_the_float64_step(t, sh, metric):
    sc = _scene()
    fl = _flags(sc, sh, metric)
    eager, act, shs = _eager(sc, t, fl)
    st, r64, r32, ref_recs = _references(sc, t, sh, metric, fl, act, shs)
    assert np.array_equal(eager["radii"], st.radii), "radii differ from the C oracle on the exported activation"
    title = f"t={t} sh={sh} metric={metric}"
    _check(f"eager {title}", eager, r64, r32, ref_recs, t)

    graph = _graphed(sc, t, fl)
    assert np.array_equal(graph["radii"], st.radii), "graph radii differ from the C oracle on the exported activation"
    vis = graph["radii"] > 0
    assert np.array_equal(graph["denom"][:, 0], vis.astype(np.float64)), "denom is not radii > 0"
    assert np.array_equal(graph["max_radii2D"], np.where(vis, graph["radii"], 0).astype(np.float64))
    _check(f"graph {title}", graph, r64, r32, ref_recs, t)


@pytest.mark.parametrize("t,sh,metric", [SCENES[0], SCENES[1]])
def test_per_splat_atomic_face_reduction_matches_the_csr_route(t, sh, metric, monkeypatch):
    """The per-face gradients summed by per-splat atomics (the C ABI's route when no CSR is given) pass the same gates
    and agree with the CSR chunk reduction."""
    from gaussianavatars_b200 import rasterizer as R
    sc = _scene()
    fl = _flags(sc, sh, metric)
    csr, act, shs = _eager(sc, t, fl)
    real = R._face_csr
    monkeypatch.setattr(R, "_face_csr", lambda binding, F, chunk=16: (real(binding, F, chunk)[0], None))
    atomic, _, _ = _eager(sc, t, fl)
    _, r64, r32, ref_recs = _references(sc, t, sh, metric, fl, act, shs)
    _check(f"atomic t={t} sh={sh} metric={metric}", atomic, r64, r32, ref_recs, t)
    a, c = atomic["grads"]["verts"], csr["grads"]["verts"]
    assert np.abs(a - c).max() <= 1e-5 * np.abs(c).max(), "dL/dverts: atomic and CSR routes differ"
    for k in fo.POSED:
        a, c = atomic["flame"][k], csr["flame"][k]
        assert np.abs(a - c).max() <= 1e-5 * np.abs(c).max(), f"dL/d{k}: atomic and CSR routes differ"
