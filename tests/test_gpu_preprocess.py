"""-m gpu: the per-splat preprocess and preprocess backward, splat by splat, read back from the frame's own scratch
(keep_last_state: the SplatRec / SplatAux records, the colour clamp bits and the g2d upstream the blend backward left),
on the edge scenes of tests/preprocess_scenes.py and a mesh-bound avatar.

* Plain route, forward: every field of every splat's record against the C oracle, bit for bit -- px, py; A', B', C'
  against the oracle's conic times REC_SCALE_* rounded in float32; opacity, rgb; radius, depth, tiles_touched (exact
  binning); the clamp bits.  Both are float32 without contraction in the same order (preprocess.cu --fmad=false, the
  oracle -ffp-contract=off).  Run with -s for each field's worst ulp distance.
* Bound route, forward: the record against the oracle fed the eager float32 activation; every conic component within
  KNIFE_CONIC_REL / 2 of the oracle's (A' and C' relative to themselves, B' to sqrt|A' C'|), except splats of the
  KNIFE_COND class: the per-component bound under which knife_edges' KNIFE_CONIC_REL Q holds.  The worst error is
  printed.  The device field-of-view route writes the same records bit for bit.
* Backward: the device's g2d row of every splat fed to the float64 VJP (dense64.project) and to the oracle's stage 5;
  every splat row of every gradient within the per-splat gate (preprocess_scenes.gate_ratio).  means2D.grad is g2d's
  first two slots exactly; culled splats and a zero upstream give exact zeros.  Printed: per tensor, p50 / p99 / max of
  the gate ratio.
"""
import numpy as np
import pytest
import torch

from oracle import binding as ob
from oracle import rasterizer as orc
from tests import adversarial_scenes as A
from tests import helpers as h
from tests import preprocess_scenes as PS

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
REC_SCALE_AC = F32(-0.5) * F32(1.4426950408889634)
REC_SCALE_B = -F32(1.4426950408889634)


@pytest.fixture(autouse=True)
def _frame_state():
    from gaussianavatars_b200 import rasterizer as R

    prev = R._EXACT_BINNING
    R.set_exact_binning(True)
    R.keep_last_state(True)
    yield
    R.keep_last_state(False)
    R.set_exact_binning(prev)


def _read(P):
    """The last training forward's records, aux, clamp bits and (after its backward) g2d rows, as numpy."""
    from gaussianavatars_b200 import rasterizer as R

    _, st, holder, _ = R._last
    assert holder is not None, "the frame was not a training forward"
    geom = h.buffer(holder, st.geom_buffer)
    offs = h.carve([48 * P, 16 * P, 4 * P, 4 * P, P, 4 * P, 4 * P, 4 * P, 4 * P, 4 * PS.G2D * P])
    f = lambda k, n: geom[offs[k]: offs[k] + n].cpu().numpy()  # noqa: E731
    aux = f(1, 16 * P).view(np.int32).reshape(P, 4)
    return dict(rec=f(0, 48 * P).view(F32).reshape(P, 12), depth=aux[:, 0].view(F32), radius=aux[:, 1],
                tiles=aux[:, 2].view(np.uint32), clamped=f(4, P), g2d=f(9, 4 * PS.G2D * P).view(F32).reshape(P, PS.G2D))


def _ulp(a, b):
    """Per-element distance in float32 ulps (ordered bit patterns)."""
    def ordered(x):
        i = np.asarray(x, F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def _unpack(bits):
    return np.stack([(bits >> ch) & 1 for ch in range(3)], 1).astype(np.uint8)


def _oracle_state(sc):
    cam = sc["cam"]
    return orc.forward(sc["means3D"].numpy(), sc["opacities"].numpy(), cam.world_view_transform.numpy(),
                       cam.full_proj_transform.numpy(), cam.camera_center.numpy(), sc["W"], sc["H"], cam.tanfovx,
                       cam.tanfovy, sc["bg"].numpy(), **PS.oracle_kwargs(sc))


def _f32_project(sc, st):
    cam = sc["cam"]
    return PS.f32_project(sc["means3D"].numpy(), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
                          sc["W"], sc["H"], cam.tanfovx, cam.tanfovy, st.cov3D)


def _report_gate(what, name, dev, ora, f64, ik, family):
    ratio = PS.assert_gate(name, dev, ora, f64, ik, family, what)
    p50, p99, worst = PS.percentiles(ratio)
    print(f"[gate] {what:<34s} dL/d{name:<15s} p50 {p50:.2e} p99 {p99:.2e} max {worst:.2e}")


ROUTES = [("shs", 3, 3, 0.7), ("shs", 1, 3, 1.0), ("colors_precomp", 0, 0, 1.0), ("cov3D_precomp", 2, 3, 1.3)]


@pytest.mark.parametrize("route", ROUTES, ids=lambda r: f"{r[0]}-deg{r[1]}of{r[2]}-mod{r[3]}")
def test_plain_route_record_and_gradients(route):
    import gaussianavatars_b200 as g

    name, deg, max_deg, mod = route
    what = f"{name}-deg{deg}of{max_deg}-mod{mod}"
    sc = PS.edge_scene(route=name, sh_degree=deg, max_sh_degree=max_deg, scale_modifier=mod)
    P, W, H = len(sc["family"]), sc["W"], sc["H"]
    st = _oracle_state(sc)
    pr = _f32_project(sc, st)
    names = [k for k in PS.PLAIN_INPUTS if k in sc and not (k == "shs" and "colors_precomp" in sc)
             and not (k in ("scales", "rotations") and "cov3D_precomp" in sc)]
    for gout_kind in ("random", "zero"):
        t = {k: sc[k].to(DEV).clone().requires_grad_(True) for k in names}
        means2D = torch.zeros((P, 3), device=DEV, requires_grad=True)
        color, radii = g.GaussianRasterizer(h.cuda_settings(sc, DEV, scale_modifier=mod))(means2D=means2D, **t)
        gen = torch.Generator().manual_seed(5)
        gout = torch.randn(3, H, W, generator=gen) if gout_kind == "random" else torch.zeros(3, H, W)
        (color * gout.to(DEV)).sum().backward()
        torch.cuda.synchronize()
        fr = _read(P)
        grads = {k: v.grad.cpu().numpy() for k, v in t.items()}
        keep = fr["radius"] > 0
        if gout_kind == "zero":
            assert not fr["g2d"].any(), "zero upstream: g2d not zero"
            for k, v in grads.items():
                assert not v.any(), f"zero upstream: dL/d{k} not exactly zero"
            assert not means2D.grad.any()
            continue

        # ---- forward: every field, bit for bit ----
        rec, con = fr["rec"], st.conic_opacity
        fields = {
            "px": (rec[:, 0], st.xy[:, 0]), "py": (rec[:, 1], st.xy[:, 1]),
            "A'": (rec[:, 2], con[:, 0] * REC_SCALE_AC), "B'": (rec[:, 3], con[:, 1] * REC_SCALE_B),
            "C'": (rec[:, 4], con[:, 2] * REC_SCALE_AC), "opacity": (rec[:, 5], np.where(keep, con[:, 3], 0)),
            "r": (rec[:, 6], st.rgb[:, 0]), "g": (rec[:, 7], st.rgb[:, 1]), "b": (rec[:, 8], st.rgb[:, 2]),
            "depth": (fr["depth"], st.depths)}
        bad = []
        for fname, (dv, ov) in fields.items():
            d = _ulp(dv, ov)
            print(f"[record] {what:<30s} {fname:<8s} worst ulp distance {int(d.max())} ({int((d > 0).sum())} splats)")
            if d.any():
                i = int(np.argmax(d))
                bad.append(f"{fname}: {int((d > 0).sum())} splats, worst splat {i} ({sc['family'][i]}) device "
                           f"{float(dv[i])!r} oracle {float(ov[i])!r}")
        for fname, dv, ov in (("radius", fr["radius"], st.radii), ("tiles", fr["tiles"], st.tiles_touched),
                              ("clamp", _unpack(fr["clamped"]), st.clamped)):
            n = int((np.asarray(dv).reshape(P, -1) != np.asarray(ov).reshape(P, -1)).any(1).sum())
            print(f"[record] {what:<30s} {fname:<8s} splats differing {n}")
            if n:
                i = int(np.nonzero((np.asarray(dv).reshape(P, -1) != np.asarray(ov).reshape(P, -1)).any(1))[0][0])
                bad.append(f"{fname}: {n} splats, first splat {i} ({sc['family'][i]}) device {dv[i]} oracle {ov[i]}")
        assert not bad, "record not bit-identical to the oracle's:\n  " + "\n  ".join(bad)
        assert not rec[~keep].any(), "a culled splat's record is not zero"

        # ---- backward: the same upstream through the float64 VJP and the oracle's stage 5 ----
        up = fr["g2d"]
        assert (means2D.grad.cpu().numpy()[:, :2] == up[:, :2]).all(), "means2D.grad differs from g2d[:, 0:2]"
        assert not up[~keep].any(), "a culled splat has a g2d row"
        clamped = _unpack(fr["clamped"])
        f64 = PS.vjp64(sc, up, keep, pr["guard"], clamped, pr["conic_dropped"])
        ora = PS.oracle_vjp(sc, st, up, radii=fr["radius"], clamped=clamped)
        ik = PS.ill_kappa_of(st, pr)
        for k, ref in f64.items():
            dev = grads[k].reshape(ref.shape)
            assert not dev.reshape(P, -1)[~keep].any(), f"dL/d{k} of a culled splat is not zero"
            _report_gate(what, k, dev, ora[k], ref, ik, sc["family"])


def _bound_inputs(sc, dtype, requires_grad):
    p = sc["params"]
    leaves = {k: p[k].to(dtype).clone().requires_grad_(requires_grad)
              for k in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")}
    b = p["binding"].long()
    fr = ob.update_mesh_properties(sc["verts"].to(dtype), sc["faces"])
    act = dict(means3D=ob.get_xyz(leaves["_xyz"], b, fr["face_center"], fr["face_orien_mat"], fr["face_scaling"]),
               scales=ob.get_scaling(leaves["_scaling"], b, fr["face_scaling"]),
               rotations=ob.get_rotation(leaves["_rotation"], b, fr["face_orien_quat"]),
               opacities=ob.get_opacity(leaves["_opacity"]),
               shs=ob.get_features(leaves["_features_dc"], leaves["_features_rest"]))
    return leaves, act, fr


@pytest.mark.parametrize("depth_alpha", [False, True], ids=["colour", "colour+alpha+depth"])
def test_bound_route_record_and_gradients(depth_alpha):
    from gaussianavatars_b200 import rasterizer as R

    sc = h.avatar_scene(P=12_000, W=320, H=240, seed=3, sh_degree=3)
    P, W, H = 12_000, sc["W"], sc["H"]
    leaves32, act32, fr32 = _bound_inputs(sc, torch.float32, True)
    sc_act = dict(sc, **{k: v.detach().contiguous() for k, v in act32.items()}, scale_modifier=1.0,
                  family=np.array(["bound"] * P))
    st = _oracle_state(sc_act)
    pr = _f32_project(sc_act, st)
    what = f"bound{'+planes' if depth_alpha else ''}"

    def frame(tanfov=None):
        t = {k: v.detach().to(DEV).requires_grad_(True) for k, v in leaves32.items()}
        face = {k: fr32[k].detach().to(DEV).contiguous() for k in ("face_center", "face_orien_mat", "face_scaling")}
        out = R.rasterize_bound(h.cuda_settings(sc, DEV), t["_xyz"], t["_rotation"], t["_scaling"], t["_opacity"],
                                t["_features_dc"], t["_features_rest"], binding=sc["params"]["binding"].to(DEV),
                                tanfov=tanfov, depth_alpha=depth_alpha, **face)
        gen = torch.Generator().manual_seed(9)
        loss = (out[0] * torch.randn(3, H, W, generator=gen).to(DEV)).sum()
        if depth_alpha:
            loss = loss + (out[2] * torch.randn(1, H, W, generator=gen).to(DEV)).sum() \
                + (out[3] * torch.randn(1, H, W, generator=gen).to(DEV)).sum()
        loss.backward()
        torch.cuda.synchronize()
        return t, _read(P)

    t, fr = frame()
    keep = fr["radius"] > 0
    rec = fr["rec"]
    # ---- forward: the conic against the oracle fed the eager activation ----
    ill = A.ill_conditioned(st) | (PS.ill_kappa_of(st, pr) > 0)
    # per component: |dA'| / |A'|, |dB'| / sqrt(|A' C'|), |dC'| / |C'|.  Within rel each, the blend's exponent moves by
    # at most 2 rel Q (|dB dx dy| <= |dB| (|A| dx^2 + |C| dy^2) / (2 sqrt|A C|)), so knife_edges' KNIFE_CONIC_REL Q
    # holds for rel <= KNIFE_CONIC_REL / 2.  (B relative to itself would be meaningless: it is ~0 for axis-aligned
    # footprints, and cancels there.)
    ref = np.stack([st.conic_opacity[:, 0] * REC_SCALE_AC, st.conic_opacity[:, 1] * REC_SCALE_B,
                    st.conic_opacity[:, 2] * REC_SCALE_AC], 1).astype(np.float64)
    size = np.stack([np.abs(ref[:, 0]), np.sqrt(np.abs(ref[:, 0] * ref[:, 2])), np.abs(ref[:, 2])], 1)
    both = keep & (st.radii > 0)
    with np.errstate(all="ignore"):
        rel = np.abs(rec[:, 2:5].astype(np.float64) - ref) / size
    worst = np.where(both, np.nan_to_num(rel, nan=np.inf).max(1), 0.0)
    bound = A.KNIFE_CONIC_REL / 2
    beyond = worst > bound
    w = float(worst[~ill].max())
    print(f"[bound record] {what}: worst conic error {w:.3e} = {w / 2.0 ** -24:.1f} x 2^-24 = {w / bound:.3f} of "
          f"KNIFE_CONIC_REL / 2 outside the KNIFE_COND class; {int(beyond.sum())} splats beyond, "
          f"{int((beyond & ill).sum())} of them KNIFE_COND ({int(both.sum())} splats compared)")
    assert not (beyond & ~ill).any(), (f"{int((beyond & ~ill).sum())} conics beyond KNIFE_CONIC_REL / 2 outside the "
                                       f"KNIFE_COND class; splat {int(np.argmax(np.where(ill, 0, worst)))}")
    assert (fr["radius"] != st.radii).sum() <= max(2, P // 2000), "radii of the bound route differ from the oracle's"
    # the device field of view writes the same records
    if not depth_alpha:
        cam = sc["cam"]
        _, fr2 = frame(torch.tensor([cam.tanfovx, cam.tanfovy], dtype=torch.float32, device=DEV))
        # (g2d is summed with float atomics in the blend backward, in no fixed order: only the records are compared)
        assert (fr2["rec"].view(np.uint32) == rec.view(np.uint32)).all(), "device-fov records differ"

    # ---- backward ----
    up = fr["g2d"]
    assert (up[:, 9] != 0).any() == depth_alpha, "the dL/dz slot is used exactly when the planes have upstream"
    clamped = _unpack(fr["clamped"])
    leaves64, act64, _ = _bound_inputs(sc, torch.float64, True)
    kw = dict(act64)
    f64 = PS.vjp64(sc_act, up, keep, pr["guard"], clamped, pr["conic_dropped"], inputs=leaves64, project_kw=kw)
    ora_act = PS.oracle_vjp(sc_act, st, up, radii=fr["radius"], clamped=clamped)
    outs = [act32[k] for k in ("means3D", "scales", "rotations", "opacities", "shs")]
    gos = [torch.from_numpy(np.ascontiguousarray(ora_act[k]).reshape(tuple(act32[k].shape)))
           for k in ("means3D", "scales", "rotations", "opacities", "shs")]
    names = list(leaves32)
    ora_leaf = torch.autograd.grad(outs, [leaves32[k] for k in names], grad_outputs=gos, allow_unused=True)
    ora = {k: (np.zeros(tuple(leaves32[k].shape)) if gr is None else gr.numpy()) for k, gr in zip(names, ora_leaf)}
    ik = PS.ill_kappa_of(st, pr)
    for k in names:
        dev = t[k].grad.cpu().numpy().reshape(f64[k].shape)
        _report_gate(what, k, dev, ora[k], f64[k], ik, sc_act["family"])
