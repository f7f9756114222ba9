"""-m gpu: FLAME posing on the device (gaussianavatars_b200.flame) against the reference -- the fixture generated from
the real FlameHead.forward / lbs (tests/golden/make_golden_flame.py) and, at full size, the float64 torch restatement
(tests/flame_oracle.py) with a self-calibrating gate: the CUDA error may be at most twice the float32 reference-order
error plus a small floor.  Then determinism, the prepared constants, and the FLAME head inside the captured training
iteration (graph.GraphedFrame) against the same iteration run eagerly."""
import os

import numpy as np
import pytest
import torch

from tests import flame_oracle as fo

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "flame_vectors.npz"))
ASSET_KEYS = ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def _g():
    import gaussianavatars_b200 as g
    return g


def _gate(what, got, ref64, ref32, floor_frac):
    """max |got - ref64| <= 2 max |ref32 - ref64| + floor_frac max |ref64|; prints both distributions."""
    got, ref64, ref32 = (np.asarray(x, np.float64) for x in (got, ref64, ref32))
    scale = float(np.abs(ref64).max()) + 1e-300
    e_c, e_32 = np.abs(got - ref64), np.abs(ref32 - ref64)
    q = lambda e: " ".join(f"{np.quantile(e, f) / scale:.2e}" for f in (0.5, 0.99, 1.0))   # noqa: E731
    print(f"[flame] {what:<34s} max|ref|={scale:.3e}  cuda p50/p99/max {q(e_c)}  fp32-oracle {q(e_32)}")
    assert np.isfinite(got).all(), what
    assert e_c.max() <= 2 * e_32.max() + floor_frac * scale, what


def _lbs(a):
    g = _g()
    return g.FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                                  a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=DEV)


def _cuda_pose(lbs, fp, t, Cw):
    """verts, verts_cano and the six gradients of sum(Cw * verts) from the CUDA operator."""
    p = {k: v.to(DEV).clone().contiguous() for k, v in fp.items() if v is not None}
    for k in fo.POSED:
        p[k].requires_grad_(True)
    verts, cano = _g().flame_pose(lbs, p, t)
    (verts * Cw).sum().backward()
    return verts.detach(), cano.detach(), {k: p[k].grad for k in fo.POSED}


def _oracle_pose(a, fp, t, Cw, dtype):
    oa = fo.assets_as({k: a[k] for k in (*ASSET_KEYS, "parents")}, dtype, DEV)
    p = {k: v.to(device=DEV, dtype=dtype).clone() for k, v in fp.items() if v is not None}
    for k in fo.POSED:
        p[k].requires_grad_(True)
    verts, cano, joints = fo.select_mesh_by_timestep(oa, p, t)
    (verts * Cw.to(dtype)).sum().backward()
    return verts.detach(), cano.detach(), {k: p[k].grad for k in fo.POSED}


def _cmp(what, cuda, o64, o32, t, floor_v=2e-6, floor_g=2e-5):
    (v, c, gr), (v64, c64, g64), (v32, c32, g32) = cuda, o64, o32
    n = lambda x: x.detach().double().cpu().numpy()   # noqa: E731
    _gate(f"{what} t={t} verts", n(v), n(v64), n(v32), floor_v)
    _gate(f"{what} t={t} verts_cano", n(c), n(c64), n(c32), floor_v)
    for k in fo.POSED:
        _gate(f"{what} t={t} d/d{k}", n(gr[k]), n(g64[k]), n(g32[k]), floor_g)
        rest = torch.cat([gr[k][:t], gr[k][t + 1:]])
        assert torch.count_nonzero(rest) == 0, f"{what}: rows other than {t} of d/d{k} are not exactly zero"


def _gold():
    a = {k: torch.tensor(GOLD[k]) for k in ASSET_KEYS}
    a.update(parents=GOLD["parents"].tolist(), faces=torch.zeros(1, 3, dtype=torch.long), n_shape=300, n_expr=100)
    fp = {k[len("param_"):]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith("param_")}
    return a, fp


def test_forward_and_backward_match_the_reference_fixture():
    a, fp = _gold()
    lbs = _lbs(a)
    T = fp["expr"].shape[0]
    for t in range(T):   # the 4 demo rows, a row with zero neck / jaw / eyes, a row near 2.5 rad
        Cw = torch.tensor(GOLD["C"][t][None], device=DEV, dtype=torch.float32)
        cuda = _cuda_pose(lbs, fp, t, Cw)
        gold = (torch.tensor(GOLD["verts"][t][None]), torch.tensor(GOLD["verts_cano"][t][None]),
                {k: torch.tensor(GOLD[f"grad_{k}"][t]) for k in fo.POSED})
        o32 = _oracle_pose(a, fp, t, Cw, torch.float32)
        _cmp("fixture", cuda, gold, o32, t)


def _full_size(T=7, seed=0):
    from gaussianavatars_b200 import synthetic as syn
    a = syn.flame_like_assets(seed)
    fp = syn.flame_like_sequence(T, seed=seed + 1, V=a["v_template"].shape[0])
    fp.pop("dynamic_offset")
    if T < 7:
        return a, fp
    g = torch.Generator().manual_seed(seed)
    for k in ("neck_pose", "jaw_pose", "eyes_pose"):
        fp[k][4] = 0.0                                                   # exactly zero (common in real tracks)
        d = torch.randn(fp[k].shape[1], generator=g)
        fp[k][5] = 1e-6 * d / d.norm()                                   # |r| ~ 1e-6
        fp[k][6] = 2.5 * d / d.norm() * (fp[k].shape[1] // 3) ** 0.5     # 2.5 rad per joint
    fp["rotation"][6] = torch.tensor([1.5, -1.8, 0.9]) * 2.5 / 2.5495
    return a, fp


def test_full_size_matches_the_float64_oracle_at_zero_small_and_large_angles():
    a, fp = _full_size()
    lbs = _lbs(a)
    V = a["v_template"].shape[0]
    gen = torch.Generator(device="cuda").manual_seed(3)
    for t in range(fp["expr"].shape[0]):
        Cw = torch.randn((1, V, 3), device=DEV, generator=gen)
        _cmp("full size", _cuda_pose(lbs, fp, t, Cw), _oracle_pose(a, fp, t, Cw, torch.float64),
             _oracle_pose(a, fp, t, Cw, torch.float32), t)


def test_gradients_are_bit_identical_run_to_run():
    a, fp = _full_size()
    lbs = _lbs(a)
    gen = torch.Generator(device="cuda").manual_seed(9)
    Cw = torch.randn((1, a["v_template"].shape[0], 3), device=DEV, generator=gen)
    for t in (2, 5):
        first = _cuda_pose(lbs, fp, t, Cw)[2]
        second = _cuda_pose(lbs, fp, t, Cw)[2]
        for k in fo.POSED:
            assert torch.equal(first[k], second[k]), f"d/d{k} differs between two identical backward calls"
            assert torch.count_nonzero(first[k][t]) > 0


def test_prepared_constants_follow_shape_and_static_offset():
    g = _g()
    a, fp = _full_size(T=4)
    lbs = _lbs(a)
    p = {k: v.to(DEV).contiguous() for k, v in fp.items()}
    Cw = torch.zeros((1, a["v_template"].shape[0], 3), device=DEV)

    def check(what):
        verts, cano = g.flame_pose(lbs, p, 1)
        o64 = _oracle_pose(a, {k: x.cpu() for k, x in p.items()}, 1, Cw, torch.float64)
        o32 = _oracle_pose(a, {k: x.cpu() for k, x in p.items()}, 1, Cw, torch.float32)
        n = lambda x: x.double().cpu().numpy()   # noqa: E731
        _gate(f"{what} verts", n(verts), n(o64[0]), n(o32[0]), 2e-6)
        _gate(f"{what} verts_cano (v_shaped)", n(cano), n(o64[1]), n(o32[1]), 2e-6)
        return verts

    v0 = check("initial shape")
    with torch.no_grad():
        p["shape"].mul_(1.7)            # in place: same tensor, new version -> re-prepared
        p["static_offset"].add_(1e-3)
    v1 = check("shape changed in place")
    assert float((v1 - v0).abs().max()) > 1e-4
    p["shape"] = p["shape"].clone()     # a new tensor object
    check("new shape tensor")
    p["shape"].requires_grad_(True)
    with pytest.raises(ValueError, match="shape"):
        g.flame_pose(lbs, p, 0)
    with pytest.raises(IndexError):
        g.flame_pose(lbs, {k: x.detach() for k, x in p.items()}, 4)


# ---- the FLAME head inside the captured iteration ----------------------------------------------------------------
W_IMG, H_IMG = 400, 304
LRS = {"xyz": 1.6e-4, "rotation": 1e-3, "scaling": 5e-3, "opacity": 5e-2, "f_dc": 2.5e-3, "f_rest": 1.25e-4}
ATTR = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")


def _flame_model(a, fp, lbs, seed=5):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    params = syn.avatar_splats(15_000, n_faces=a["faces"].shape[0], seed=seed, sh_degree=3, scale_gain=2.5)
    p = {k: v.to(DEV).clone().contiguous() for k, v in fp.items()}
    pc = MeshBoundGaussians(params, 3, None, None, device=DEV, requires_grad=True, flame=lbs, flame_param=p)
    for attr in ATTR:
        setattr(pc, attr, torch.nn.Parameter(getattr(pc, attr).detach().clone()))
    return pc


def _scene():
    from gaussianavatars_b200 import synthetic as syn
    a, fp = _full_size(T=6, seed=2)
    cam = syn.orbit_camera(W_IMG, H_IMG, r=1.0, fovy_deg=20.0, azimuth_deg=15.0)
    gt = torch.randint(0, 256, (3, H_IMG, W_IMG), generator=torch.Generator().manual_seed(7), dtype=torch.uint8).to(DEV)
    return a, fp, cam, gt


def _eager_frame(pc, t, cam, gt):
    g = _g()
    from gaussianavatars_b200.renderer import render
    for x in pc.parameters() + [pc.flame_param[k] for k in fo.POSED]:
        x.grad = None
    pc.select_mesh_by_timestep(t)
    out = render(cam.to(DEV), pc, Pipe, torch.ones(3, device=DEV))
    loss = g.photometric_loss(out["render"], gt, 0.2)
    lx, ls = g.binding_regularizers(pc._xyz, pc._scaling, out["radii"], pc.binding, pc.face_scaling)
    total = loss + lx + ls
    total.backward()
    return out["render"].detach(), total.detach(), [p.grad.clone() for p in pc.parameters()], \
        {k: pc.flame_param[k].grad.clone() for k in fo.POSED}


def _close(a, b, what, rtol=2e-5):   # gradients differ only by the atomic summation order of the splat backward
    scale = float(b.abs().max()) + 1e-30
    d = float((a - b).abs().max())
    assert d <= rtol * scale, f"{what}: max diff {d:.3e} vs max|ref| {scale:.3e}"


def test_graphed_frame_poses_the_flame_head_per_timestep_without_recapture():
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    g = _g()
    a, fp, cam, gt = _scene()
    pc = _flame_model(a, fp, _lbs(a))
    pc_e = _flame_model(a, fp, _lbs(a))
    for k in fo.POSED:
        pc.flame_param[k].requires_grad_(True)
        pc_e.flame_param[k].requires_grad_(True)
    fr = GraphedFrame(pc, W_IMG, H_IMG, cam.FoVx, cam.FoVy, torch.ones(3), loss="photometric", regularizers={})
    fr.set_inputs(camera=camera_block(cam).to(DEV), gt_u8=gt, timestep=0)
    with pytest.raises(ValueError, match="timestep"):
        fr.set_inputs(verts=torch.zeros(a["v_template"].shape[0], 3, device=DEV))
    with pytest.raises(IndexError):
        fr.set_inputs(timestep=6)
    for t in (0, 1, 2, 3, 2, 1, 0):
        fr.set_inputs(timestep=t)
        fr.run(check=True)
        torch.cuda.synchronize()
        img, loss, grads, fgrads = _eager_frame(pc_e, t, cam, gt)
        assert torch.equal(fr.image, img), f"t={t}: image differs from the eager frame"
        assert abs(float(fr.loss) - float(loss)) <= 1e-6 * abs(float(loss)), t
        for p, q in zip(pc.parameters(), grads):
            _close(p.grad, q, f"t={t} splat gradient")
        for k in fo.POSED:
            _close(pc.flame_param[k].grad, fgrads[k], f"t={t} d/d{k}", rtol=1e-4)
            assert torch.count_nonzero(torch.cat([pc.flame_param[k].grad[:t], pc.flame_param[k].grad[t + 1:]])) == 0
    assert fr.captures == 1, "changing the timestep must not re-capture"
    with torch.no_grad():
        pc.flame_param["shape"].mul_(1.1)   # a changed shape is baked into the prepared constants: re-capture
    fr.run(check=True)
    assert fr.captures == 2


def test_full_flame_training_iteration_in_one_graph_matches_the_eager_iteration():
    """8 iterations: capturable Adam over the splat groups and the reference's FLAME groups, densification statistics
    on, in one replay each -- against the eager iteration with the FLAME pose from the float32 reference-order oracle,
    torch's Adam on the FLAME groups and the host-stepped Adam on the splats."""
    from types import SimpleNamespace
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    from gaussianavatars_b200.renderer import render
    g = _g()
    a, fp, cam, gt = _scene()
    pc = _flame_model(a, fp, _lbs(a))
    fgroups = g.flame_param_groups(pc.flame_param)
    groups = [{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pc.parameters())]
    opt = g.Adam(groups + fgroups, lr=0.0, eps=1e-15, capturable=True)
    P = pc._xyz.shape[0]
    for n in ("xyz_gradient_accum", "denom"):
        setattr(pc, n, torch.zeros((P, 1), device=DEV))
    pc.max_radii2D = torch.zeros((P,), device=DEV)
    fr = GraphedFrame(pc, W_IMG, H_IMG, cam.FoVx, cam.FoVy, torch.ones(3), loss="photometric", regularizers={},
                      optimizer=opt, densify_stats=True)
    fr.set_inputs(camera=camera_block(cam).to(DEV), gt_u8=gt, timestep=0)

    # eager twin: the same initial state, FLAME from the oracle
    pe = _flame_model(a, fp, _lbs(a))
    oa = fo.assets_as({k: a[k] for k in (*ASSET_KEYS, "parents")}, torch.float32, DEV)
    opt_s = g.Adam([{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pe.parameters())], lr=0.0, eps=1e-15)
    opt_f = torch.optim.Adam(g.flame_param_groups(pe.flame_param), lr=0.0, eps=1e-15)
    for n in ("xyz_gradient_accum", "denom"):
        setattr(pe, n, torch.zeros((P, 1), device=DEV))
    pe.max_radii2D = torch.zeros((P,), device=DEV)
    f0 = {k: pe.flame_param[k].detach().clone() for k in fo.POSED}
    steps = [0, 1, 2, 3, 1, 0, 2, 3]
    for i, t in enumerate(steps):
        fr.set_inputs(timestep=t)
        fr.run(check=True)
        opt_s.zero_grad(set_to_none=True)
        opt_f.zero_grad(set_to_none=True)
        verts, _, _ = fo.select_mesh_by_timestep(oa, pe.flame_param, t)
        pe.update_mesh_properties(verts[0])
        out = render(cam.to(DEV), pe, Pipe, torch.ones(3, device=DEV))
        loss = g.photometric_loss(out["render"], gt, 0.2)
        lx, ls = g.binding_regularizers(pe._xyz, pe._scaling, out["radii"], pe.binding, pe.face_scaling)
        (loss + lx + ls).backward()
        g.add_densification_stats(pe, SimpleNamespace(grad=out["viewspace_points"].grad), out["radii"])
        opt_s.step()
        opt_f.step()
        torch.cuda.synchronize()
        rel = abs(float(fr.loss) - float((loss + lx + ls))) / abs(float(loss + lx + ls))
        print(f"[flame-train] step {i} t={t} loss graph {float(fr.loss):.7f} eager {float(loss + lx + ls):.7f} rel {rel:.1e}")
        assert rel <= 1e-4, f"step {i}: loss differs"
    assert fr.captures == 1 and not fr.overflowed()
    for k in fo.POSED:
        dg = (pc.flame_param[k].detach() - f0[k]).cpu()
        de = (pe.flame_param[k].detach() - f0[k]).cpu()
        assert torch.count_nonzero(dg[4:]) == 0 and torch.count_nonzero(de[4:]) == 0, "unvisited rows moved"
        assert torch.count_nonzero(dg[:4]) > 0
        err = float((dg - de).abs().max()) / (float(de.abs().max()) + 1e-30)
        print(f"[flame-train] {k:<12s} max|step sum| {float(de.abs().max()):.3e}  graph vs eager {err:.2e} of it")
        assert err <= 0.05, k
    for n, p, q in zip(LRS, pc.parameters(), pe.parameters()):
        d = (p.detach() - q.detach()).abs()
        bound = 2 * len(steps) * LRS[n]          # Adam moves an entry by at most ~lr per step
        frac = float((d > 0.25 * bound).float().mean())
        print(f"[flame-train] {n:<9s} max|diff| {float(d.max()):.2e} (Adam bound {bound:.1e}) frac>bound/4 {frac:.1e}")
        assert frac <= 1e-2, n
    for n in ("denom", "max_radii2D"):
        assert torch.equal(getattr(pc, n), getattr(pe, n)) or \
            float((getattr(pc, n) != getattr(pe, n)).float().mean()) <= 1e-3, n
    assert float(opt.state[pc.flame_param["expr"]]["step"]) == len(steps)
