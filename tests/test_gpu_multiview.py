"""-m gpu: every camera of a rig in one forward (gab200_forward_views, render_views, the K-view GraphedRender and
GraphedEval).

The K views are one frame of K * P virtual splats; the per-splat depth sort restricted to one view is that view's own
order and tiles of different views are disjoint, so every output must equal K single-camera forwards
(gab200_forward_display with each camera's device field of view) bit for bit: torch.equal, no tolerance."""
import ctypes as C

import pytest
import torch

from tests import helpers as h
from tests.test_gpu_camera_fov import _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


@pytest.fixture(autouse=True)
def default_policies():
    """Culled binning, the default tile sort and the LATE policy around every test (all process-wide)."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    prev = R._EXACT_BINNING
    knob = N.tune(N.TUNE_TILE_SORT)
    yield
    R.set_exact_binning(prev)
    N.tune(N.TUNE_TILE_SORT, knob)
    R.set_sync_policy("late")


def _table(cams, blind=(), bad_fov=()):
    """(K,37) device table of the cameras; rows in `blind` look away from the scene, rows in `bad_fov` carry an
    invalid tan(FoV/2)."""
    from gaussianavatars_b200.renderer import camera_table
    t = camera_table(cams, DEV)
    for k in blind:   # the scene lies behind this camera: nothing passes the near plane
        wv = t[k, :16].view(4, 4).clone()
        wv[3, 2] = -50.0   # world_view_transform is stored transposed: [3, 2] is the z translation
        t[k, :16] = wv.reshape(-1)
    for k, v in zip(bad_fov, (0.0, float("nan"), -1.0, float("inf"))):
        t[k, 35 + (k % 2)] = v
    return t.contiguous()


def _base_args(sc, kind, colors):
    """ForwardArgs of the scene (P, image, inputs), camera fields left to the caller, and the tensors they point at."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200.rasterizer import face_frame
    rs = h.cuda_settings(sc, DEV, debug=False)
    a = N.ForwardArgs()
    if kind == "bound":
        p = sc["params"]
        P = p["_xyz"].shape[0]
        keep = list(R._fill_common(a, rs, DEV, P, False))
        a.input_mode = N.INPUT_BOUND_RAW
        leaves = [p[k].to(DEV).contiguous() for k in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc",
                                                       "_features_rest")]
        fc, fR, fs = face_frame(sc["verts"].to(DEV), sc["faces"].to(DEV))
        binding = p["binding"].to(DEV).to(torch.int32).contiguous()
        keep += leaves + [fc, fR, fs, binding]
        a.means3D, a.rotations, a.scales, a.opacities = (t.data_ptr() for t in leaves[:4])
        a.sh_dc, a.sh_rest = leaves[4].data_ptr(), leaves[5].data_ptr()
        a.sh_coeffs = 1 + leaves[5].shape[1]
        a.binding, a.num_faces = binding.data_ptr(), fc.shape[0]
        a.face_center, a.face_orien_mat, a.face_scaling = fc.data_ptr(), fR.data_ptr(), fs.data_ptr()
    else:
        P = sc["means3D"].shape[0]
        keep = list(R._fill_common(a, rs, DEV, P, False))
        a.input_mode = N.INPUT_ACTIVATED
        ts = [sc[k].to(DEV).contiguous() for k in ("means3D", "opacities", "scales", "rotations", "shs")]
        keep += ts
        a.means3D, a.opacities, a.scales, a.rotations = (t.data_ptr() for t in ts[:4])
        a.shs, a.sh_coeffs = ts[4].data_ptr(), ts[4].shape[1]
    if colors:
        g = torch.Generator().manual_seed(5)
        col = torch.rand((P, 3), generator=g).to(DEV)
        keep.append(col)
        a.colors_precomp = col.data_ptr()
        if kind != "bound":
            a.shs, a.sh_coeffs = None, 0
    a.exact_binning = int(R._EXACT_BINNING)
    return a, keep, P


def _copy(a):
    from gaussianavatars_b200 import _native as N
    b = N.ForwardArgs()
    C.pointer(b)[0] = a
    return b


def _single(a, table, k, W, H):
    """View k through gab200_forward_display (EXACT): float image, bytes, radii, visibility."""
    import gaussianavatars_b200.rasterizer as R
    b = _copy(a)
    row = table[k]
    b.viewmatrix, b.projmatrix, b.campos = row.data_ptr(), row[16:].data_ptr(), row[32:].data_ptr()
    rgb8 = torch.empty((H, W, 3), dtype=torch.uint8, device=DEV)
    R.set_sync_policy("exact")
    color, radii, st, _ = R._run_forward(b, DEV, False, R.FrameHints(), row[35:37], rgb8, True)
    vis = R.visible_of(radii).clone()
    torch.cuda.synchronize()
    return color.clone(), rgb8, radii.clone(), vis, st


def _views(a, table, W, H, sync="exact", capacity=0, depth=(0, 0), outputs="both"):
    """One gab200_forward_views call in a sync mode: (color, bytes, radii, visibility, state, n, flag)."""
    from gaussianavatars_b200 import _native as N
    K, P = table.shape[0], a.P
    b = _copy(a)
    b.viewmatrix = b.projmatrix = b.campos = None
    color = torch.full((K, 3, H, W), -7.0, device=DEV) if outputs != "u8" else None
    rgb8 = torch.full((K, H, W, 3), 7, dtype=torch.uint8, device=DEV) if outputs != "float" else None
    radii = torch.full((K, P), -7, dtype=torch.int32, device=DEV)
    vis = torch.zeros((K, P), dtype=torch.bool, device=DEV)
    b.out_color, b.radii, b.visibility = N.ptr(color), radii.data_ptr(), vis.data_ptr()
    holder = []

    def alloc(user, nbytes):
        t = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=DEV)
        holder.append(t)
        return t.data_ptr()
    cb = N.ALLOC_FN(alloc)
    b.alloc_geom = b.alloc_binning = b.alloc_image = cb
    counters = torch.zeros(N.NUM_COUNTERS, dtype=torch.int32).pin_memory()
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    b.sync_mode = {"exact": N.SYNC_EXACT, "late": N.SYNC_LATE, "none": N.SYNC_NONE}[sync]
    b.binning_hint = capacity
    b.depth_hint_lo, b.depth_hint_hi = depth
    b.frame_seq = 3
    b.counters_host, b.overflow_flag = counters.data_ptr(), flag.data_ptr()
    st = N.FrameState()
    n = N.lib().gab200_forward_views(C.byref(b), K, table.data_ptr(), N.ptr(rgb8), C.byref(st),
                                     C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    N.check(n, "gab200_forward_views")
    torch.cuda.synchronize()
    return color, rgb8, radii, vis, st, n, int(flag.item())


def _check(a, table, W, H, singles=None, **kw):
    """gab200_forward_views in the given mode against the K single-view forwards; returns them and the K-view state."""
    K = table.shape[0]
    singles = singles or [_single(a, table, k, W, H) for k in range(K)]
    color, rgb8, radii, vis, st, n, flag = _views(a, table, W, H, **kw)
    assert flag == 0, f"{kw}: the overflow flag is set"
    outputs = kw.get("outputs", "both")
    for k, (c1, u1, r1, v1, _) in enumerate(singles):
        if outputs != "u8":
            assert torch.equal(color[k], c1), f"{kw}: view {k} float image differs"
        if outputs != "float":
            assert torch.equal(rgb8[k], u1), f"{kw}: view {k} display bytes differ"
        assert torch.equal(radii[k], r1), f"{kw}: view {k} radii differ"
        assert torch.equal(vis[k], v1), f"{kw}: view {k} visibility differs"
    if kw.get("sync", "exact") != "none":
        assert n == sum(int(s[4].num_rendered) for s in singles), "the K-view frame's instances are the views' sum"
    return singles, st


def _depth_range(singles):
    lo = min(int(s[4].depth_key_min) for s in singles if s[4].depth_key_min <= s[4].depth_key_max)
    hi = max(int(s[4].depth_key_max) for s in singles if s[4].depth_key_min <= s[4].depth_key_max)
    return lo, hi


@pytest.mark.parametrize("tile_sort", [0, 1])
@pytest.mark.parametrize("exact_binning", [False, True])
def test_views_equal_single_view_forwards_in_every_mode(exact_binning, tile_sort):
    """K = 1 and 3, ragged image size, distinct FoVs, a camera that sees nothing and one with an invalid tan(FoV):
    EXACT, LATE with a capacity far too small, NONE with room; no depth hint, a fitting hint and one that overflows a
    bucket; the float image only, the bytes only and both."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    R.set_exact_binning(exact_binning)
    N.tune(N.TUNE_TILE_SORT, tile_sort)
    sc = h.avatar_scene(P=12_000, W=333, H=250, seed=4)
    a, keep, P = _base_args(sc, "bound", False)
    cams = _rig(333, 250, n=5)
    for table in (_table(cams[:1]), _table(cams[1:4]), _table(cams, blind=(1,), bad_fov=(3,))):
        singles, st = _check(a, table, 333, 250)
        n = int(st.num_rendered)
        assert n > 10_000
        for k, s in enumerate(singles):
            if table.shape[0] == 5 and k in (1, 3):
                assert int((s[2] > 0).sum()) == 0 and torch.equal(s[1], s[1][:1, :1].expand_as(s[1]))
            else:
                assert int((s[2] > 0).sum()) > 1000, "view renders nothing"
        lo, hi = _depth_range(singles)
        _check(a, table, 333, 250, singles, sync="late", capacity=1024)
        _check(a, table, 333, 250, singles, sync="late", capacity=n + 100, depth=(lo, hi))
        _check(a, table, 333, 250, singles, sync="none", capacity=n + 100, depth=(lo, hi))
        _, st2 = _check(a, table, 333, 250, singles, sync="exact", depth=(hi - 2, hi - 1))   # every key in one bucket
        assert st2.depth_sort_path == 2 and st2.attempts == 2, "the overflowing hint did not take the radix path"
        _check(a, table, 333, 250, singles, outputs="float")
        _check(a, table, 333, 250, singles, sync="late", capacity=1024, outputs="u8")
    del keep


def test_none_mode_raises_the_sticky_flag_on_overflow():
    sc = h.avatar_scene(P=12_000, W=320, H=240, seed=4)
    a, keep, P = _base_args(sc, "bound", False)
    table = _table(_rig(320, 240, n=3))
    *_, n, flag = _views(a, table, 320, 240, sync="none", capacity=4096)
    assert flag == 1
    del keep


@pytest.mark.parametrize("kind,colors", [("activated", False), ("activated", True), ("bound", True)])
def test_views_with_activated_inputs_and_precomputed_colours(kind, colors):
    sc = h.random_scene(P=10_000, W=301, H=211, sh_degree=3, seed=4) if kind == "activated" else \
        h.avatar_scene(P=12_000, W=301, H=211, seed=4)
    a, keep, P = _base_args(sc, kind, colors)
    from gaussianavatars_b200 import synthetic as syn
    base = sc["cam"]
    cams = [syn.look_at_camera(301, 211, 50.0 + 4 * i, 38.0 + 3 * i, w2c=base.world_view_transform.T.numpy())
            for i in range(3)] if kind == "activated" else _rig(301, 211, n=3)
    singles, _ = _check(a, _table(cams), 301, 211)
    assert all(int((s[2] > 0).sum()) > 1000 for s in singles)
    _check(a, _table(cams), 301, 211, singles, sync="late", capacity=1024)
    del keep


@pytest.mark.parametrize("tile_sort", [0, 1])
def test_sixteen_views_at_1080p_with_long_tile_lists(tile_sort):
    """16 cameras at 1920x1080, 100k splats plus a stack of 3000 copies of one splat: its tiles' lists are beyond the
    shared-memory tile sort (2048 entries: the counting sort's bitmap path)."""
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    N.tune(N.TUNE_TILE_SORT, tile_sort)
    sc = h.avatar_scene(P=100_000, W=1920, H=1080, seed=4)
    p = sc["params"]
    stack = 3000
    for k in p:   # splat 0 repeated: identical keys, ties broken by id
        p[k] = torch.cat([p[k], p[k][:1].expand(stack, *p[k].shape[1:])]).contiguous()
    a, keep, P = _base_args(sc, "bound", False)
    cams = _rig(1920, 1080, n=16)
    table = _table(cams)
    singles, st = _check(a, table, 1920, 1080)
    R.keep_last_state(True)
    try:
        _single(a, table, 0, 1920, 1080)
        _, _, ranges, _ = R.export_last_binning()
    finally:
        R.keep_last_state(False)
    assert int((ranges[:, 1] - ranges[:, 0]).max()) > 2048, "no tile list beyond the shared-memory sort"
    _check(a, table, 1920, 1080, singles, sync="late", capacity=1024)
    # no depth hint: the 16 x 3000 stacked copies share one depth per view, more than a depth bucket holds
    _check(a, table, 1920, 1080, singles, sync="none", capacity=int(st.num_rendered) + 100)
    del keep


# ---- Python surface and graphs --------------------------------------------------------------------------------------
def _flame_setup(T=8):
    from tests.test_gpu_flame import _flame_model, _full_size, _lbs
    a, fp = _full_size(T=T, seed=2)
    return _flame_model(a, fp, _lbs(a))


W_IMG, H_IMG = 400, 304


def test_render_views_equals_render_display():
    from gaussianavatars_b200.renderer import camera_table, render_display, render_views
    pc = _flame_setup()
    pc.select_mesh_by_timestep(3)
    cams = [c.to(DEV) for c in _rig(W_IMG, H_IMG, n=4)]
    bg = torch.tensor([0.2, 0.5, 0.9], device=DEV)
    out = render_views(cams, pc, Pipe, bg, float_image=True)
    assert out["display_u8"].shape == (4, H_IMG, W_IMG, 3) and out["render"].shape == (4, 3, H_IMG, W_IMG)
    for k, cam in enumerate(cams):
        ref = render_display(cam, pc, Pipe, bg, float_image=True)
        for key in ("display_u8", "render", "radii", "visibility_filter"):
            assert torch.equal(out[key][k], ref[key]), f"view {k}: {key} differs"
    tab = render_views(camera_table(cams, DEV), pc, Pipe, bg, width=W_IMG, height=H_IMG)
    assert tab["render"] is None and torch.equal(tab["display_u8"], out["display_u8"])


def test_graphed_render_k_views_equals_render_views_without_recapture():
    from gaussianavatars_b200.graph import GraphedRender
    from gaussianavatars_b200.renderer import render_views
    pc = _flame_setup()
    cams = [c.to(DEV) for c in _rig(W_IMG, H_IMG, n=8)]
    groups = [cams[:4], cams[4:]]
    bg = torch.tensor([1.0, 1.0, 1.0])
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", host_slots=2, views_per_replay=4, warm_cameras=groups,
                         warm_timesteps=range(8))
    hosts = []
    for i, t in enumerate((0, 5, 2, 7)):
        view.set_inputs(cameras=groups[i % 2], timestep=t)
        view.run(check=True)
        pc.select_mesh_by_timestep(t)
        ref = render_views(groups[i % 2], pc, Pipe, bg.to(DEV), float_image=True)
        torch.cuda.synchronize()
        assert torch.equal(view.image, ref["render"]) and torch.equal(view.display, ref["display_u8"])
        assert torch.equal(view.radii, ref["radii"]), f"replay {i}: radii differ"
        hosts.append(ref["display_u8"].cpu())
    assert view.captures == 1 and view.display.shape == (4, H_IMG, W_IMG, 3)
    assert torch.equal(view.host_frame(3), hosts[3]) and torch.equal(view.host_frame(2), hosts[2])
    with pytest.raises(IndexError):
        view.host_frame(1)


def test_graphed_eval_k_views_equals_single_view_rows_and_skips_overflowed_replays():
    from gaussianavatars_b200.graph import GraphedEval
    pc = _flame_setup()
    cams = [c.to(DEV) for c in _rig(W_IMG, H_IMG, n=6)]
    bg = torch.tensor([1.0, 1.0, 1.0])
    g = torch.Generator().manual_seed(3)
    gts = torch.randint(0, 256, (6, 3, H_IMG, W_IMG), generator=g, dtype=torch.uint8).to(DEV)
    steps = (1, 6)
    for source in ("float", "u8"):
        one = GraphedEval(pc, W_IMG, H_IMG, bg, views=6, source=source, warm_cameras=cams, warm_timesteps=steps)
        many = GraphedEval(pc, W_IMG, H_IMG, bg, views=6, source=source, views_per_replay=3,
                           warm_cameras=[cams[:3], cams[3:]], warm_timesteps=steps)
        for grp in range(2):
            t = steps[grp]
            for k in range(3):
                i = 3 * grp + k
                one.set_inputs(camera=cams[i], timestep=t, gt_u8=gts[i], view=i)
                one.run(check=True)
            many.set_inputs(cameras=cams[3 * grp:3 * grp + 3], timestep=t, gt_u8=gts[3 * grp:3 * grp + 3],
                            view=3 * grp)
            many.run(check=True)
        a, b = one.scores(), many.scores()
        assert torch.equal(a["per_view"], b["per_view"]), f"{source}: K-view rows differ from single-view rows"
        assert many.captures == 1

    # a replay whose capacity is far too small writes none of its rows
    small = GraphedEval(pc, W_IMG, H_IMG, bg, views=6, views_per_replay=3, capacity=2048,
                        warm_cameras=[cams[:3]], warm_timesteps=steps)
    small.set_inputs(cameras=cams[3:], timestep=1, gt_u8=gts[3:], view=3)
    small.run()
    assert small.overflowed()
    assert torch.isnan(small.table[3:]).all() and torch.isnan(small.table[:3]).all()
    with pytest.raises(RuntimeError, match="hold no score"):
        small.scores()
