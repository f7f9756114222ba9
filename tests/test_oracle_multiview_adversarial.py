"""CPU: the mesh-bound camera rigs of tests/bound_rigs.py put each adversarial scene at the edges they exist for, in the
views meant to reach them.

The float32 C oracle runs per view on the activation of oracle/binding.py's getters.  Asserted per rig: the binding
reproduces the scene within a few ulps and is as lopsided as promised; the narrowed view has splats outside its guard
band that are inside view 0's and still reach the image; the dolly culls a band at the near plane that view 0 draws,
and the mirrored view draws splats view 0 culls there; SH degree 3 colours clamp in one view and not in another;
stacks stay beyond 2048 entries in every valid view; faint pairs sit on both sides of 1/255 in every valid view.
tests/test_gpu_multiview_adversarial.py relies on these regimes; a rig that loses one fails here first."""
import numpy as np
import pytest
import torch

from oracle import binding as ob
from oracle import rasterizer as orc
from tests import adversarial_scenes as A
from tests import bound_rigs as B

MAIN = ["needles", "near_plane", "guard_band", "saturating_stack", "faint", "tile_borders+ties", "guard_band+sh3"]
CASES = [(n, None, None) for n in MAIN] + [(n, W, H) for (W, H) in A.RAGGED_SIZES for n in A.BUILDERS]


def _cid(c):
    return c[0] if c[1] is None else f"{c[0]}-{c[1]}x{c[2]}"


def scene(case):
    """The activated scene of a case: the builders of tests/adversarial_scenes.py; the main saturating stack also
    holds a 2100-splat stack (beyond the 1984 / 2048 blend thresholds)."""
    name, W, H = case
    if name.startswith("walk:"):      # the walk scenes of tests/walk_scenes.py
        from tests import walk_scenes as WS
        return WS.build(name[5:])
    if name == "saturating_stack" and W is None:
        sc = A.saturating_stack(stacks=(20, 400, 2100))
        sc["name"] = name
        return sc
    return A.build(name, W, H)


def oracle_views(bound, act, K=6):
    """The C oracle per valid view of the rig on the activation `act` (None for the invalid-FoV view)."""
    n = lambda t: t.detach().float().numpy()   # noqa: E731
    out = []
    for k, cam in enumerate(B.rig(bound, K)):
        if not B.valid(k):
            out.append(None)
            continue
        out.append(orc.forward(n(act["means3D"]), n(act["opacities"]), cam.world_view_transform.numpy(),
                               cam.full_proj_transform.numpy(), cam.camera_center.numpy(), bound["W"], bound["H"],
                               cam.tanfovx, cam.tanfovy, bound["bg"].numpy(), shs=n(act["shs"]),
                               sh_degree=bound["sh_degree"], scales=n(act["scales"]), rotations=n(act["rotations"])))
    return out


def regime_counts(bound, means3D, sts):
    """What a six-view rig reaches, from the oracle's per-view state (`means3D`: the activation the states were
    computed on)."""
    cams = B.rig(bound, 6)
    m = np.asarray(means3D, np.float32)
    r = [None if s is None else s.radii for s in sts]
    d0, d2 = B.view_depth(cams[0], m), B.view_depth(cams[2], m)
    both_vis_clamp_diff = 0
    for a in range(5):
        for c in range(a + 1, 5):
            both = (r[a] > 0) & (r[c] > 0)
            both_vis_clamp_diff += int((sts[a].clamped[both] != sts[c].clamped[both]).sum())
    faint = []
    for s in sts[:5]:
        t = A.pair_table(s)
        near = (t["power"] <= 0) & (np.abs(t["alpha"].astype(np.float64) * 255.0 - 1.0) < 1e-3)
        acc = t["alpha"] >= A.ALPHA_MIN
        faint.append((int((near & acc).sum()), int((near & ~acc).sum())))
    return dict(
        guard0=int((B.guard_out(cams[0], m) & (r[0] > 0)).sum()),
        guard_narrow=int((B.guard_out(cams[1], m) & (r[1] > 0) & ~B.guard_out(cams[0], m)).sum()),
        dolly_culled=int(((d2 <= np.float32(0.2)) & (r[2] == 0) & (r[0] > 0)).sum()),
        mirror_shows=int(((d0 <= np.float32(0.2)) & (r[0] == 0) & (r[3] > 0)).sum()),
        clamp_differs=both_vis_clamp_diff,
        max_list=[int((s.ranges[:, 1].astype(np.int64) - s.ranges[:, 0]).max()) for s in sts[:5]],
        faint=faint,
        radius0_k3=int(np.all([x == 0 for x in r[:3]], axis=0).sum()),
        visible=[int((x > 0).sum()) for x in r[:5]])


def _ulps(got, ref, mag):
    d = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    return float((d / np.spacing(np.asarray(mag, np.float32)).astype(np.float64)).max()) if d.size else 0.0


@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_bound_rig_reaches_its_regimes(case):
    sc = scene(case)
    bound = B.bind(sc)
    p = bound["params"]
    P = p["_xyz"].shape[0]
    # the binding: lopsided, empty faces, neighbours on different faces, both kinds of face in use
    b = p["binding"].long()
    F = bound["faces"].shape[0]
    counts = torch.bincount(b, minlength=F).numpy()
    assert (counts == 0).sum() >= 3, "no empty faces"
    if P > 74:
        assert counts.max() > 64, "no face with more than 64 splats"
    if P >= 12:
        assert np.unique(b.numpy()).size >= 2 and bound["exact"][np.unique(b.numpy())].any() and \
            (~bound["exact"][np.unique(b.numpy())]).any(), "splats are not on both kinds of face"
    # the round trip through the getters, in float32: a few ulps (means: of the larger of the mean and its face centre)
    act, _, _ = B.activate(bound)
    s = bound["scene"]
    fr = ob.update_mesh_properties(bound["verts"], bound["faces"])
    mag = np.maximum(np.abs(s["means3D"].numpy()).max(1), np.abs(fr["face_center"][b].numpy()).max(1))
    e_mean = _ulps(act["means3D"].detach(), s["means3D"], mag[:, None])
    e_scale = _ulps(act["scales"].detach(), s["scales"], s["scales"].numpy())
    e_op = _ulps(act["opacities"].detach(), s["opacities"], s["opacities"].numpy())
    q, q0 = act["rotations"].detach().double(), s["rotations"].double()
    q = q * torch.sign((q * q0).sum(1, keepdim=True))
    e_rot = _ulps(q, q0, np.ones_like(q0.numpy()))
    assert torch.equal(act["shs"].detach(), s["shs"])
    print(f"[round-trip] {_cid(case):<26s} ulps: mean {e_mean:.1f} scale {e_scale:.1f} opacity {e_op:.1f} "
          f"rotation {e_rot:.1f}")
    # exp of a rounded log: the scale's error is the rounding of _scaling (|_scaling| up to ~10) times the scale
    assert max(e_mean, e_op, e_rot) <= 4.0 and e_scale <= 8.0, "the binding does not reproduce the scene"

    sts = oracle_views(bound, act)
    c = regime_counts(bound, act["means3D"].detach().numpy(), sts)
    print(f"[regimes] {_cid(case):<26s} P={P} " + " ".join(f"{k}={v}" for k, v in c.items()))
    name = case[0]
    if name == "near_plane":
        assert c["dolly_culled"] >= 10, "the dolly culls no band at the near plane"
        assert c["mirror_shows"] >= 4, "the mirrored view shows none of view 0's near-culled splats"
        assert c["radius0_k3"] >= 1, "no splat with radius 0 in each of the first three views"
    if case[1] is None:
        if name in ("needles", "near_plane", "saturating_stack"):
            assert c["guard_narrow"] >= (1 if name == "near_plane" else 10), \
                "the narrowed view puts no visible splat outside its guard band"
        if name.startswith("guard_band"):
            assert c["guard0"] >= 20, "view 0 has too few visible splats beyond its guard band"
        if name == "guard_band+sh3":
            assert c["clamp_differs"] >= 20, "no colour channel clamps in one view and not in another"
        if name == "saturating_stack":
            assert min(c["max_list"]) > 2048, "a valid view lost the stack beyond 2048 entries"
        if name == "faint":
            assert all(a >= 3 and r >= 3 for a, r in c["faint"]), "a valid view lacks faint pairs on both sides"
    # every view with an invalid field of view is skipped; every valid one draws something
    assert all(v > 0 for v in c["visible"])
