"""-m gpu: the CUDA path against the CPU oracle on the adversarial scenes (tests/adversarial_scenes.py), under every
schedule the sort and the blend can run in.

Schedule matrix (full cross product, 24 schedules; every test of this file runs under each):
    GAB200_TUNE_TILE_SORT   0 cub radix | 1 counting
    GAB200_TUNE_DEPTH_SORT  0 bucket (needs a depth hint: the compared frame is the second one) | 1 radix
    binning                 exact | culled
    blend                   default | HEAVY_FWD = 1984 (forward light wherever allowed) | HEAVY_BWD = 32 (backward K = 2
                            on every tile of 32 or more entries)
Per scene and schedule: radii bit-exact; the sorted stream bit-exact (exact binning) or an order-preserving
subsequence keeping every instance the oracle's blend accepted (culled); image and final_T within the parity budget
and the image bit-identical across all schedules; every input gradient within the explained gate
(helpers.assert_grad_explained: no entry beyond the tolerance outside adversarial_scenes.knife_edges) of the oracle's
and of the first schedule's, exactly zero for splats without an instance and for clamped colour channels; on the ragged sizes
the display bytes equal render.py's quantisation, and (first schedule) image and gradients equal float64 autograd of
the dense model."""
import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import helpers as h

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SCHEDULES = [(ts, ds, exact, blend) for ts in (0, 1) for ds in (0, 1) for exact in (True, False)
             for blend in ("default", "fwd1984", "bwd32")]
MAIN = ["needles", "near_plane", "guard_band", "saturating_stack", "faint", "tile_borders+ties", "guard_band+sh3"]
CASES = [(n, None, None) for n in MAIN] + [(n, W, H) for (W, H) in A.RAGGED_SIZES for n in A.BUILDERS]


def _cid(c):
    return c[0] if c[1] is None else f"{c[0]}-{c[1]}x{c[2]}"


def _sid(s):
    return f"tile{'radix' if s[0] == 0 else 'count'}-depth{'bucket' if s[1] == 0 else 'radix'}-" \
           f"{'exact' if s[2] else 'culled'}-{s[3]}"


@pytest.fixture(autouse=True, params=SCHEDULES, ids=_sid)
def schedule(request):
    """Sets the knobs of one schedule and restores every previous value afterwards (GAB200_TEST_TUNE runs keep theirs
    for the rest of the suite; the "default" blend leaves the heavy thresholds as they are)."""
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import rasterizer as R

    ts, ds, exact, blend = request.param
    knobs = {N.TUNE_TILE_SORT: ts, N.TUNE_DEPTH_SORT: ds}
    if blend == "fwd1984":
        knobs[N.TUNE_HEAVY_FWD] = 1984
    elif blend == "bwd32":
        knobs[N.TUNE_HEAVY_BWD] = 32
    prev = {k: N.tune(k, v) for k, v in knobs.items()}
    prev_exact = R._EXACT_BINNING
    R.set_exact_binning(exact)
    R.keep_last_state(True)
    yield request.param
    R.set_exact_binning(prev_exact)
    for k, v in prev.items():
        N.tune(k, v)


_REF = {}      # case -> oracle forward / backward and what the checks derive from them
_FIRST = {}    # case -> (schedule, image, gradients) of the first schedule that ran it


def _scene(case):
    name, W, H = case
    if name == "saturating_stack" and W is None:
        sc = A.saturating_stack(stacks=(20, 400, 2100))   # 2100 > the 1984 / 2048 heavy thresholds
        sc["name"] = name
        return sc
    return A.build(name, W, H)


def _reference(case):
    if case not in _REF:
        sc = _scene(case)
        st = h.oracle_forward(sc)
        gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(7))
        g = h.oracle_backward(sc, st, gout.numpy())
        ke = A.knife_edges(st)
        print(f"[knife] {_cid(case)}: {ke['pairs']} pairs, {int(ke['pixels'].sum())} pixels, "
              f"{int(ke['splats'].sum())}/{st.P} splats")
        _REF[case] = dict(sc=sc, st=st, gout=gout, g=g, accepted=A.accepted_instances(st), ke=ke)
    return _REF[case]


def _inputs(sc, grad):
    t = {k: sc[k].to(DEV).clone().requires_grad_(grad) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    t["means2D"] = torch.zeros((sc["means3D"].shape[0], 3), device=DEV, requires_grad=grad)
    return t


def _forward(rasterizer, t, **over):
    kw = dict(means3D=t["means3D"], means2D=t["means2D"], opacities=t["opacities"], shs=t["shs"], scales=t["scales"],
              rotations=t["rotations"])
    kw.update(over)
    return rasterizer(**kw)


def _run(sc, sched, gout):
    """The compared frame of one schedule: with the bucket depth sort, a first frame leaves the depth hint behind and
    the second frame is the one that counts."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import rasterizer as R

    hints = R.FrameHints()
    rs = h.cuda_settings(sc, DEV)
    if sched[1] == 0:
        with torch.no_grad():
            _forward(g.GaussianRasterizer(rs, hints), _inputs(sc, False))
    t = _inputs(sc, True)
    img, radii = _forward(g.GaussianRasterizer(rs, hints), t)
    torch.cuda.synchronize()
    keys, vals, ranges, n = R.export_last_binning()
    info = R.last_frame_info()
    out = dict(img=img.detach().clone(), radii=radii.cpu().numpy(), n=n, path=info["depth_sort_path"],
               keys=keys.cpu().numpy().view(np.uint64), vals=vals.cpu().numpy().view(np.uint32),
               ranges=ranges.cpu().numpy().view(np.uint32))
    (img * gout.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    out["grads"] = {k: t[k].grad.cpu().numpy() for k in ("means3D", "means2D", "opacities", "scales", "rotations", "shs")}
    # final_T: black splats over a white background render T itself
    white = dict(sc, bg=torch.ones(3))
    with torch.no_grad():
        tw = _inputs(sc, False)
        imgT, _ = _forward(g.GaussianRasterizer(h.cuda_settings(white, DEV), R.FrameHints()), tw, shs=None,
                           colors_precomp=torch.zeros_like(tw["means3D"]))
    out["T"] = imgT.cpu().numpy()
    return out


def _display(sc):
    """gab200_forward_display on the activated inputs: (float image, display bytes) of one forward."""
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import rasterizer as R

    t = _inputs(sc, False)
    rs = h.cuda_settings(sc, DEV, debug=False)
    a = N.ForwardArgs()
    keep = R._fill_common(a, rs, DEV, t["means3D"].shape[0], False)
    a.input_mode = N.INPUT_ACTIVATED
    a.sh_coeffs = t["shs"].shape[1]
    a.means3D, a.opacities, a.shs = t["means3D"].data_ptr(), t["opacities"].data_ptr(), t["shs"].data_ptr()
    a.scales, a.rotations = t["scales"].data_ptr(), t["rotations"].data_ptr()
    rgb8 = torch.full((sc["H"], sc["W"], 3), 7, dtype=torch.uint8, device=DEV)
    img, *_ = R._run_forward(a, DEV, False, R.FrameHints(), None, rgb8, True)
    torch.cuda.synchronize()
    del keep
    return img, rgb8


def _quant(img):
    """render.py's conversion of the float image."""
    return img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_adversarial_scene(case, schedule):
    ref = _reference(case)
    sc, st, g_ref, ke = ref["sc"], ref["st"], ref["g"], ref["ke"]
    what = f"{_cid(case)} [{_sid(schedule)}]"
    out = _run(sc, schedule, ref["gout"])

    # 1. radii
    assert np.array_equal(out["radii"], st.radii), f"{what}: radii differ from the oracle"
    if schedule[1] == 0 and (st.radii > 0).any():
        assert out["path"] != 0, f"{what}: the hinted frame did not take the bucket depth sort"
    # 2. sorted stream
    if schedule[2]:
        assert out["n"] == st.N, f"{what}: {out['n']} instances, oracle {st.N}"
        assert np.array_equal(out["keys"], st.keys_sorted), f"{what}: sorted tile|depth keys not bit-exact"
        assert np.array_equal(out["vals"], st.vals_sorted), f"{what}: sorted splat ids not bit-exact"
        assert np.array_equal(out["ranges"], st.ranges), f"{what}: tile ranges differ"
    else:
        full = {(int(k), int(v)): i for i, (k, v) in enumerate(zip(st.keys_sorted, st.vals_sorted))}
        missing = [(int(k), int(v)) for k, v in zip(out["keys"], out["vals"]) if (int(k), int(v)) not in full]
        assert not missing, f"{what}: culled stream has instances the oracle's list does not: {missing[:4]}"
        pos = np.array([full[(int(k), int(v))] for k, v in zip(out["keys"], out["vals"])], np.int64)
        assert (np.diff(pos) > 0).all(), f"{what}: culled stream is not an order-preserving subsequence"
        dropped = np.setdiff1d(ref["accepted"], pos)
        assert dropped.size == 0, (f"{what}: culling dropped {dropped.size} instances the oracle's blend accepted, e.g. "
                                   f"tile {st.keys_sorted[dropped[0]] >> np.uint64(32)} splat {st.vals_sorted[dropped[0]]}")
    # 3. image
    img = out["img"].cpu().numpy()
    s = h.image_stats(img, st.out_color)
    print(f"[image] {what:<60s} max|d|={s['max_abs']:.3e} >1e-4: {s['n_over_1e4']}/{s['n']}")
    h.assert_image_explained(img, st.out_color, ke["pixels"], f"{what}: image")
    # 4. final_T
    h.assert_image_explained(out["T"], np.broadcast_to(st.final_T, out["T"].shape), ke["pixels"], f"{what}: final_T")
    # 5. gradients
    for k, g in out["grads"].items():
        h.assert_grad_explained(g, g_ref[k], A.affected(ke, k), f"{_cid(case)} dL/d{k}")
    invis = st.radii == 0
    for k, g in out["grads"].items():
        assert not np.any(g[invis]), f"{what}: dL/d{k} nonzero for a splat without an instance"
    clamped = st.clamped.astype(bool)                                        # (P, 3)
    gsh = out["grads"]["shs"]                                                # (P, M, 3)
    assert not np.any(gsh.transpose(0, 2, 1)[clamped]), f"{what}: SH gradient through a clamped colour channel"
    nb = (sc["sh_degree"] + 1) ** 2
    assert not np.any(gsh[:, nb:]), f"{what}: gradient of an unused SH coefficient"
    # across schedules: the same image bit for bit, gradients within the same gate
    first = _FIRST.setdefault(case, (schedule, out["img"], out["grads"]))
    assert torch.equal(out["img"], first[1]), f"{what}: image differs from schedule [{_sid(first[0])}]"
    for k, g in out["grads"].items():
        h.assert_grad_explained(g, first[2][k], A.affected(ke, k), f"{_cid(case)} dL/d{k} vs first schedule")
    if case[1] is None:
        return
    # 6. display bytes (ragged sizes)
    img_d, rgb8 = _display(sc)
    assert torch.equal(img_d, out["img"]), f"{what}: display forward's float image differs"
    assert torch.equal(rgb8, _quant(img_d)), f"{what}: display bytes differ from render.py's quantisation"
    # 7. float64 anchor (first schedule only: every schedule equals it above)
    if first[0] == schedule:
        from tests.test_oracle_adversarial import dense_image_and_grads

        img64, g64 = dense_image_and_grads(sc, st, seed=7)
        h.assert_image_explained(img, img64, ke["pixels"], f"{what}: image vs float64")
        for k, g in out["grads"].items():
            h.assert_grad_explained(g, g64[k], A.affected(ke, k), f"{_cid(case)} dL/d{k} vs float64")
