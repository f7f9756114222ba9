"""-m gpu: the K-view training frame (rasterize_bound_views_train: gab200_forward_views_train, gab200_backward_views) on
the mesh-bound adversarial rigs of tests/bound_rigs.py, where one splat sits at a different edge in each view.

Cases and schedules (the 24 schedules of tests/test_gpu_adversarial.py: tile sort x depth sort with its two-frame
hint x exact / culled binning x default / HEAVY_FWD = 1984 / HEAVY_BWD = 32):
    main cases (needles, near_plane, guard_band, saturating_stack with a 2100 stack, faint, tile_borders+ties,
    guard_band+sh3)                                     K = 3 under all 24 schedules; K = 1, 2, 6 under the first
    the six builders at the ragged sizes                K = 6 under the first schedule and under
                                                        tile count / depth radix / culled / HEAVY_BWD = 32
Per case, K and schedule:
    forward     images, radii and visibility equal K single-view rasterize_bound forwards (each with its own tanfov)
                bit for bit, and the first schedule's images; radii equal the C oracle on the exported activation;
                images within the parity budget of the oracle
    singles     summed raw gradients, dL/dverts and each view's dL/dmeans2D row against K single-view steps summed
    oracle      the same against the C-oracle backward per view, pulled back through oracle/binding.py in float64
    float64     (ragged, first schedule) the same against oracle/dense64.py per view pinned to that view's oracle
                decisions, through float64 binding autograd
    zeros       radius 0 in every view -> zero raw gradients; radius 0 in a view -> zero dL/dmeans2D row; the
                invalid-FoV view -> culled, background, zero row; a channel clamped wherever visible -> zero SH
                gradient; unused SH coefficients -> zero; the repeated view -> view 0's image bit for bit and its
                dL/dmeans2D row under the gate
Raw and means2D gradients are held to helpers.assert_grad_tight, dL/dverts to train_step_oracle.gate_vertex."""

import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import bound_rigs as B
from tests import helpers as h
from tests import train_step_oracle as T
from tests import walk_scenes as WS
from tests.test_oracle_multiview_adversarial import MAIN, scene

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SCHEDULES = [(ts, ds, exact, blend) for ts in (0, 1) for ds in (0, 1) for exact in (True, False)
             for blend in ("default", "fwd1984", "bwd32")]
FIRST = SCHEDULES[0]
RAGGED_SECOND = (1, 1, False, "bwd32")
RAGGED = [(n, W, H) for (W, H) in A.RAGGED_SIZES for n in A.BUILDERS]


def _cid(c):
    return c[0] if c[1] is None else f"{c[0]}-{c[1]}x{c[2]}"


def _sid(s):
    return f"tile{'radix' if s[0] == 0 else 'count'}-depth{'bucket' if s[1] == 0 else 'radix'}-" \
           f"{'exact' if s[2] else 'culled'}-{s[3]}"


@pytest.fixture
def schedule(request):
    """Sets the knobs of one schedule and restores every previous value afterwards (sync policy and the kept state
    included; GAB200_TEST_TUNE runs keep theirs: the "default" blend leaves the heavy thresholds as they are)."""
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import rasterizer as R

    ts, ds, exact, blend = request.param
    knobs = {N.TUNE_TILE_SORT: ts, N.TUNE_DEPTH_SORT: ds}
    if blend == "fwd1984":
        knobs[N.TUNE_HEAVY_FWD] = 1984
    elif blend == "bwd32":
        knobs[N.TUNE_HEAVY_BWD] = 32
    prev = {k: N.tune(k, v) for k, v in knobs.items()}
    prev_exact, prev_policy = R._EXACT_BINNING, R._SYNC_POLICY
    R.set_exact_binning(exact)
    yield request.param
    R.set_exact_binning(prev_exact)
    R.set_sync_policy(prev_policy)
    for k, v in prev.items():
        N.tune(k, v)


# ---- per case: the rig, the exported activation, the C oracle per view ---------------------------------------------
_CASE = {}     # case -> bound rig, activation, oracle states and backward per view
_SINGLE = {}   # (case, view) -> one single-view step of this library
_FIRST = {}    # (case, K) -> (schedule, images) of the first schedule that ran it
_DENSE = {}    # (case, K) -> float64 gradients summed over the views


def _settings(bound, row=None):
    from gaussianavatars_b200.rasterizer import GaussianRasterizationSettings
    bg = bound["bg"].to(DEV)
    if row is None:
        return GaussianRasterizationSettings(bound["H"], bound["W"], 1.0, 1.0, bg, 1.0, None, None,
                                             bound["sh_degree"], None, False, False)
    return GaussianRasterizationSettings(bound["H"], bound["W"], 1.0, 1.0, bg, 1.0, row[:16].clone(),
                                         row[16:32].clone(), bound["sh_degree"], row[32:35].clone(), False, False)


def _dpix(bound, view):
    """dL/dimage of one view; the repeated view (4) takes view 0's."""
    seed = 0 if view == 4 else view
    g = torch.Generator().manual_seed(100 + seed)
    return torch.randn((3, bound["H"], bound["W"]), generator=g)


def _leaves(bound):
    p = bound["params"]
    leaves = {k: p[k].to(DEV).clone().requires_grad_(True) for k in B.RAW}
    verts = bound["verts"].to(DEV).clone().requires_grad_(True)
    return leaves, verts


def _case(case):
    if case in _CASE:
        return _CASE[case]
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.rasterizer import face_frame
    from oracle import rasterizer as orc
    bound = B.bind(scene(case))
    p = bound["params"]
    with torch.no_grad():
        fc, fR, fs = face_frame(bound["verts"].to(DEV), bound["faces"].to(DEV))
        act = [t.cpu() for t in g.bind_activate(1.0, p["_xyz"].to(DEV), p["_rotation"].to(DEV),
                                                p["_scaling"].to(DEV), p["_opacity"].to(DEV), p["binding"].to(DEV),
                                                fc, fR, fs)]
    means3D, opac, _, cov = (t.numpy() for t in act)
    shs = torch.cat([p["_features_dc"], p["_features_rest"]], 1).numpy()
    cams = B.rig(bound, 6)
    fl = dict(sh_degree=bound["sh_degree"], bg=bound["bg"].numpy())
    sts, gs = [], []
    for k, cam in enumerate(cams):
        if not B.valid(k):
            sts.append(None)
            gs.append(None)
            continue
        st = T.oracle_forward_on(act[0], act[1], cam, bound["W"], bound["H"], fl, torch.from_numpy(shs), cov3D=act[3])
        gk = orc.backward(st, _dpix(bound, k).numpy(), means3D, cam.world_view_transform.numpy(),
                          cam.full_proj_transform.numpy(), cam.camera_center.numpy(), cam.tanfovx, cam.tanfovy,
                          bound["bg"].numpy(), shs=shs, sh_degree=bound["sh_degree"])
        sts.append(st)
        gs.append(gk)
    _CASE[case] = dict(bound=bound, cams=cams, sts=sts, gs=gs, act=act)
    return _CASE[case]


def _single(case, view):
    """One single-view training step of this library (rasterize_bound with the view's own tanfov) for view `view`."""
    key = (case, view)
    if key in _SINGLE:
        return _SINGLE[key]
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound, visible_of
    c = _case(case)
    bound = c["bound"]
    row = B.table(c["cams"], DEV)[view]
    leaves, verts = _leaves(bound)
    fc, fR, fs = face_frame(verts, bound["faces"].to(DEV))
    P = leaves["_xyz"].shape[0]
    m2d = torch.zeros((P, 3), device=DEV, requires_grad=True)
    color, radii = rasterize_bound(_settings(bound, row), *(leaves[k] for k in B.RAW),
                                   bound["params"]["binding"].to(DEV), fc, fR, fs, means2D=m2d,
                                   tanfov=row[35:37].clone())
    vis = visible_of(radii).clone()
    (color * _dpix(bound, view).to(DEV)).sum().backward()
    torch.cuda.synchronize()
    z = lambda t, like: (t if t is not None else torch.zeros_like(like)).double().cpu().numpy()  # noqa: E731
    _SINGLE[key] = dict(img=color.detach().clone(), radii=radii.clone(), vis=vis,
                        grads={k: z(leaves[k].grad, leaves[k]) for k in B.RAW}, verts=z(verts.grad, verts),
                        m2d=m2d.grad.double().cpu().numpy())
    return _SINGLE[key]


def _views(case, K, sched):
    """One K-view training frame; with the bucket depth sort a first frame leaves the depth hint behind and the
    second is the one compared."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound_views_train, visible_of
    c = _case(case)
    bound = c["bound"]
    table = B.table(c["cams"][:K], DEV)
    dpix = torch.stack([_dpix(bound, k) for k in range(K)]).to(DEV)
    hints = R.FrameHints()
    P = bound["params"]["_xyz"].shape[0]

    def frame(train):
        leaves, verts = _leaves(bound)
        fc, fR, fs = face_frame(verts, bound["faces"].to(DEV))
        m2d = torch.zeros((K, P, 3), device=DEV, requires_grad=True)
        color, radii = rasterize_bound_views_train(_settings(bound), table, *(leaves[k] for k in B.RAW),
                                                   bound["params"]["binding"].to(DEV), fc, fR, fs, means2D=m2d,
                                                   hints=hints)
        if not train:
            return None
        vis = visible_of(radii).clone()
        (color * dpix).sum().backward()
        torch.cuda.synchronize()
        return dict(img=color.detach().clone(), radii=radii.clone(), vis=vis,
                    grads={k: leaves[k].grad.double().cpu().numpy() for k in B.RAW},
                    verts=verts.grad.double().cpu().numpy(), m2d=m2d.grad.double().cpu().numpy(),
                    path=hints.last["depth_sort_path"])
    if sched[1] == 0:
        frame(False)
    return frame(True)


def _pull_back(bound, act, leaves, verts, outputs, grads):
    got = torch.autograd.grad(outputs, [leaves[k] for k in B.RAW] + [verts], grads, allow_unused=True)
    z = lambda t, like: (t if t is not None else torch.zeros_like(like)).numpy()  # noqa: E731
    return {k: z(t, leaves[k]) for k, t in zip(B.RAW, got[:-1])}, z(got[-1], verts)


def _reference32(case, K):
    """The reference's own float32 chain, summed over the valid views among the first K: the float32 getters of
    oracle/binding.py, the C oracle per view on their scales and rotations (its float32 dL/dSigma -> scale, rotation),
    float32 autograd back to the raw parameters."""
    from oracle import rasterizer as orc
    c = _case(case)
    bound = c["bound"]
    act, leaves, verts = B.activate(bound, torch.float32, requires_grad=True)
    n = {k: act[k].detach().numpy() for k in ("means3D", "opacities", "scales", "rotations", "shs")}
    fl = dict(sh_degree=bound["sh_degree"], bg=bound["bg"].numpy())
    sums = {k: 0.0 for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    for k, cam in enumerate(c["cams"][:K]):
        if not B.valid(k):
            continue
        st = T.oracle_forward_on(act["means3D"], act["opacities"], cam, bound["W"], bound["H"], fl, act["shs"],
                                 scales=act["scales"], rotations=act["rotations"])
        gk = orc.backward(st, _dpix(bound, k).numpy(), n["means3D"], cam.world_view_transform.numpy(),
                          cam.full_proj_transform.numpy(), cam.camera_center.numpy(), cam.tanfovx, cam.tanfovy,
                          bound["bg"].numpy(), shs=n["shs"], sh_degree=bound["sh_degree"], scales=n["scales"],
                          rotations=n["rotations"])
        for key in sums:
            sums[key] = sums[key] + gk[key]
    outputs = [act[k] for k in sums]
    grads = [torch.as_tensor(np.asarray(v, np.float32)).reshape(o.shape) for v, o in zip(sums.values(), outputs)]
    return _pull_back(bound, act, leaves, verts, outputs, grads)


def _oracle_sum(case, K, dtype=torch.float64):
    """The C oracle's per-view backward summed over the valid views among the first K, pulled back through the
    getters of oracle/binding.py in float64."""
    c = _case(case)
    bound = c["bound"]
    act, leaves, verts = B.activate(bound, dtype, requires_grad=True)
    gs = [g for g in c["gs"][:K] if g is not None]
    P = leaves["_xyz"].shape[0]
    if not gs:
        return {k: np.zeros(leaves[k].shape) for k in B.RAW}, np.zeros(verts.shape)
    s = lambda k: torch.from_numpy(sum(np.asarray(g[k], np.float64) for g in gs)).to(dtype)  # noqa: E731
    outputs = [act["means3D"], act["cov3D"], act["opacities"], act["shs"]]
    grads = [s("means3D"), s("cov3D_precomp"), s("opacities").reshape(P, 1), s("shs")]
    return _pull_back(bound, act, leaves, verts, outputs, grads)


def _dense_sum(case, K):
    """oracle/dense64.py per valid view among the first K, pinned to that view's oracle decisions, through float64
    binding autograd, summed."""
    key = (case, K)
    if key in _DENSE:
        return _DENSE[key]
    from oracle import dense64
    c = _case(case)
    bound = c["bound"]
    act, leaves, verts = B.activate(bound, torch.float64, requires_grad=True)
    P = leaves["_xyz"].shape[0]
    # values pinned to the exported float32 activation, derivatives of the float64 chain: a splat the float32 path puts
    # at z = 0.2f (just in front of the near plane) must not land on 0.2 in float64 and drop out
    pinned = {k: v + (torch.as_tensor(e).to(torch.float64).reshape(v.shape) - v).detach()
              for (k, v), e in zip(((k, act[k]) for k in ("means3D", "opacities", "cov3D")), (c["act"][0], c["act"][1],
                                                                                                c["act"][3]))}
    total = torch.zeros((), dtype=torch.float64)
    m2ds = []
    d = torch.float64
    for k in range(K):
        m2 = torch.zeros(P, 3, dtype=d, requires_grad=True)
        m2ds.append(m2)
        st = c["sts"][k]
        if st is None:
            continue
        pin = T.pin_of(st)
        idx = torch.nonzero(torch.from_numpy(pin["radii"]) > 0).reshape(-1)
        if idx.numel() == 0:
            continue
        cam = c["cams"][k]
        img, _ = dense64.render(pinned["means3D"][idx], m2[idx], pinned["opacities"][idx],
                                cam.world_view_transform.to(d), cam.full_proj_transform.to(d), cam.camera_center.to(d),
                                bound["W"], bound["H"], cam.tanfovx, cam.tanfovy, bound["bg"].to(d),
                                shs=act["shs"][idx], sh_degree=bound["sh_degree"], cov3D_precomp=pinned["cov3D"][idx],
                                radii=torch.from_numpy(pin["radii"]).long()[idx],
                                rect_xy=torch.from_numpy(pin["xy"])[idx], depths=torch.from_numpy(pin["depths"])[idx])
        total = total + (img * _dpix(bound, k).to(d)).sum()
    leaf_list = [leaves[k] for k in B.RAW] + [verts] + m2ds
    got = torch.autograd.grad(total, leaf_list, allow_unused=True) if total.requires_grad else [None] * len(leaf_list)
    z = lambda t, like: (t if t is not None else torch.zeros_like(like)).detach().numpy()  # noqa: E731
    out = ({k: z(t, leaves[k]) for k, t in zip(B.RAW, got[:6])}, z(got[6], verts),
           [z(t, m) for t, m in zip(got[7:], m2ds)])
    _DENSE[key] = out
    return out


def _gate_all(what, got, raw, verts, m2d_rows, K, slack, kes):
    """Summed raw gradients and each valid view's dL/dmeans2D row under assert_grad_explained (the knife set of a raw
    gradient is the union of the valid views' knife_edges; of a view's row, that view's), dL/dverts under
    train_step_oracle.gate_vertex.  An array the fixed gate rejects passes only if its largest error stays within
    `slack` of it: twice the error of the reference's own float32 chain (_reference32) against the float64 one, the
    rule of test_gpu_train_step.  A needle's covariance has a condition number near 1e6, and any float32 route from
    the image to its scale and rotation -- the reference's, or the same sums taken in another order -- loses digits
    the fixed gate would ask for."""
    def fallback(name, a, ref):
        e_c = float(np.abs(np.asarray(a, np.float64) - ref).max())
        print(f"[grad] {what} {name} beyond the fixed gate: max|d| {e_c:.3e}, 2 x float32 reference {slack[name]:.3e}")
        assert e_c <= slack[name], f"{what}: {name} beyond the gate and beyond twice the float32 reference's error"
    live = [ke for ke in kes if ke is not None]
    for k in B.RAW:
        aff = np.zeros(got["grads"][k].shape[0], bool)
        for ke in live:
            aff |= A.affected(ke, k)
        try:
            h.assert_grad_explained(got["grads"][k], raw[k], aff, f"{what} d{k}")
        except AssertionError:
            fallback(k, got["grads"][k], raw[k])
    rec = T.gate_vertex(f"{what} dverts", got["verts"], verts)
    print(f"[grad] {what + ' dverts':<28s} n={rec['n']:>9d} worst={rec['worst']:.2e} outliers={rec['outliers']}/"
          f"{rec['allowed']}")
    if not rec["ok"]:
        fallback("verts", got["verts"], verts)
    for k in range(K):
        if m2d_rows[k] is not None:
            aff = np.zeros(m2d_rows[k].shape[0], bool) if kes[k] is None else A.affected(kes[k], "means2D")
            h.assert_grad_explained(got["m2d"][k], m2d_rows[k], aff, f"{what} dmeans2D view {k}")


def _check(case, K, sched):
    c = _case(case)
    bound = c["bound"]
    what = f"{_cid(case)} K={K} [{_sid(sched)}]"
    out = _views(case, K, sched)
    singles = [_single(case, k) for k in range(K)]
    P = bound["params"]["_xyz"].shape[0]
    kes = [None if st is None else A.knife_edges(st) for st in c["sts"][:K]]
    print(f"[knife] {what}: " + ", ".join("-" if ke is None else f"{int(ke['pixels'].sum())} px/{int(ke['splats'].sum())} "
                                          f"splats" for ke in kes))
    if sched[1] == 0 and any(s is not None and (s.radii > 0).any() for s in c["sts"][:K]):
        assert out["path"] != 0, f"{what}: the hinted frame did not take the bucket depth sort"

    # 1. forward: K single views bit for bit, the first schedule's images, the oracle's radii and image
    for k in range(K):
        s = singles[k]
        assert torch.equal(out["img"][k], s["img"]), f"{what}: view {k} image differs from its single-view forward"
        assert torch.equal(out["radii"][k], s["radii"]), f"{what}: view {k} radii differ from the single view's"
        assert torch.equal(out["vis"][k], s["vis"]), f"{what}: view {k} visibility differs from the single view's"
        st = c["sts"][k]
        radii = out["radii"][k].cpu().numpy()
        if st is None:
            assert not radii.any(), f"{what}: the invalid-FoV view kept a splat"
            bg = bound["bg"].to(DEV)[:, None, None].expand(3, bound["H"], bound["W"])
            assert torch.equal(out["img"][k], bg), f"{what}: the invalid-FoV view is not the background"
            continue
        assert np.array_equal(radii, st.radii), f"{what}: view {k} radii differ from the C oracle"
        h.assert_image_explained(out["img"][k].cpu().numpy(), st.out_color, kes[k]["pixels"],
                                 f"{what}: view {k} image vs oracle")
    first = _FIRST.setdefault((case, K), (sched, out["img"]))
    assert torch.equal(out["img"], first[1]), f"{what}: images differ from schedule [{_sid(first[0])}]"

    # the reference's float32 chain against its float64 one: the slack of an array the fixed gate rejects
    raw_o, verts_o = _oracle_sum(case, K)
    raw_32, verts_32 = _reference32(case, K)
    slack = {k: 2 * float(np.abs(np.asarray(raw_32[k], np.float64) - raw_o[k]).max()) for k in B.RAW}
    slack["verts"] = 2 * float(np.abs(np.asarray(verts_32, np.float64) - verts_o).max())

    # 2. against K single-view steps, summed
    raw = {k: sum(s["grads"][k] for s in singles) for k in B.RAW}
    _gate_all(f"{_cid(case)} K={K} vs singles", out, raw, sum(s["verts"] for s in singles),
              [s["m2d"] for s in singles], K, slack, kes)

    # 3. against the C oracle per view, pulled back in float64
    _gate_all(f"{_cid(case)} K={K} vs oracle", out, raw_o, verts_o,
              [None if g is None else g["means2D"] for g in c["gs"][:K]], K, slack, kes)

    # 4. against float64 (ragged sizes, first schedule)
    if case[1] is not None and sched == FIRST:
        raw_d, verts_d, m2d_d = _dense_sum(case, K)
        _gate_all(f"{_cid(case)} K={K} vs float64", out, raw_d, verts_d,
                  [None if c["sts"][k] is None else m2d_d[k] for k in range(K)], K, slack, kes)

    # 5. exact zeros
    radii = out["radii"].cpu().numpy()                                        # (K, P)
    dark = (radii == 0).all(0)
    for k in B.RAW:
        assert not out["grads"][k][dark].any(), f"{what}: d{k} nonzero for a splat with radius 0 in every view"
    assert not out["m2d"][radii == 0].any(), f"{what}: a dL/dmeans2D row nonzero in a view where the radius is 0"
    for k in range(K):
        if c["sts"][k] is None:
            assert not out["m2d"][k].any(), f"{what}: the invalid-FoV view wrote dL/dmeans2D"
    # a channel clamped in every view where the splat is visible: no SH gradient on it
    seen = radii > 0
    always = np.ones((P, 3), bool)
    for k in range(K):
        if c["sts"][k] is not None:
            always &= np.where(seen[k][:, None], c["sts"][k].clamped.astype(bool), True)
    always &= seen.any(0)[:, None]
    gsh = np.concatenate([out["grads"]["_features_dc"], out["grads"]["_features_rest"]], 1)   # (P, M, 3)
    assert not gsh.transpose(0, 2, 1)[always].any(), f"{what}: SH gradient through a channel clamped in every view"
    nb = (bound["sh_degree"] + 1) ** 2
    assert gsh.shape[1] > nb or bound["sh_degree"] == 3
    assert not gsh[:, nb:].any(), f"{what}: gradient of an unused SH coefficient"
    if K > 4:
        assert torch.equal(out["img"][4], out["img"][0]), f"{what}: the repeated view's image differs from view 0's"
        h.assert_grad_tight(out["m2d"][4], out["m2d"][0], f"{_cid(case)} K={K} dmeans2D view 4 vs 0")
    print(f"[zeros] {what}: dark {int(dark.sum())}/{P}, rows of radius 0 {int((radii == 0).sum())}, "
          f"channels clamped wherever visible {int(always.sum())}")


@pytest.mark.parametrize("schedule", SCHEDULES, ids=_sid, indirect=True)
@pytest.mark.parametrize("case", [(n, None, None) for n in MAIN], ids=_cid)
def test_main_cases_three_views_every_schedule(case, schedule):
    _check(case, 3, schedule)


@pytest.mark.parametrize("schedule", [FIRST], ids=_sid, indirect=True)
@pytest.mark.parametrize("K", [1, 2, 6])
@pytest.mark.parametrize("case", [(n, None, None) for n in MAIN], ids=_cid)
def test_main_cases_other_view_counts(case, K, schedule):
    _check(case, K, schedule)


@pytest.mark.parametrize("schedule", [FIRST, RAGGED_SECOND], ids=_sid, indirect=True)
@pytest.mark.parametrize("case", RAGGED, ids=_cid)
def test_ragged_sizes_six_views(case, schedule):
    _check(case, 6, schedule)


@pytest.mark.parametrize("schedule", [FIRST, (0, 1, True, "bwd32")], ids=_sid, indirect=True)
@pytest.mark.parametrize("case", [("walk:" + n, None, None) for n in WS.WALK], ids=_cid)
def test_walk_scenes_six_views(case, schedule):
    """The walk scenes bound to a rig: a K-view backward whose global tile order interleaves the views
    (tests/test_oracle_walk.py), light-only and with K = 2 on every tile of 32 or more entries."""
    _check(case, 6, schedule)
