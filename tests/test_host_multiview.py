"""CPU: the multi-view forward -- the gab200_forward_views entry point (export, ctypes signature, the argument checks
that reject before any device work) and the host-side checks of render_views, rasterize_bound_views and the K-view
GraphedRender / GraphedEval -- no compute calls (no GPU)."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMMY = 0x1000   # never dereferenced: every call below is rejected during argument validation


def test_forward_views_is_exported_with_the_header_signature():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    assert "gab200_forward_views" in N.EXPORTED_SYMBOLS and hasattr(L, "gab200_forward_views")
    f = L.gab200_forward_views
    assert f.restype is C.c_int64
    assert f.argtypes == [C.POINTER(N.ForwardArgs), C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(N.FrameState),
                          C.c_void_p]
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    m = re.search(r"int64_t gab200_forward_views\(([^)]*)\);", hdr)
    assert m, "gab200_forward_views is not declared in the header"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert params == ["const gab200_forward_args* args", "int32_t views", "const float* cameras", "uint8_t* out_rgb8",
                      "gab200_frame_state* state_out", "void* stream"]
    assert re.search(r"#define GAB200_CAMERA_FLOATS 37\b", hdr) and N.CAMERA_FLOATS == 37
    assert L.gab200_abi_version() == N.ABI_VERSION == 3   # a new entry point, the argument struct is unchanged


def _args(P=0, W=33, H=17, need_backward=0, out_color=DUMMY):
    from gaussianavatars_b200 import _native as N

    a = N.ForwardArgs()
    a.abi_version, a.input_mode, a.P = N.ABI_VERSION, N.INPUT_BOUND_RAW, P
    a.image_width, a.image_height = W, H
    a.need_backward = need_backward
    a.bg = DUMMY   # viewmatrix / projmatrix / campos stay NULL: the camera table replaces them
    a.out_color = out_color
    a.alloc_geom = a.alloc_binning = a.alloc_image = N.ALLOC_CALLBACK
    if P > 0:
        a.means3D = a.opacities = a.scales = a.rotations = a.sh_dc = a.radii = DUMMY
        a.sh_coeffs, a.sh_degree = 1, 0
    return a


@pytest.mark.parametrize("case", ["views0", "views_negative", "views_too_many", "cameras_null", "state_null",
                                  "args_null", "need_backward", "no_output", "bad_abi", "views_times_P",
                                  "views_times_tiles", "missing_splat_input"])
def test_forward_views_rejects_bad_arguments_before_any_device_work(case):
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    st = N.FrameState()
    a, views, cams, rgb8, state = _args(), 2, DUMMY, DUMMY, C.byref(st)
    if case == "views0":
        views = 0
    elif case == "views_negative":
        views = -3
    elif case == "views_too_many":
        views = N.MAX_VIEWS + 1
    elif case == "cameras_null":
        cams = None
    elif case == "state_null":
        state = None
    elif case == "need_backward":
        a = _args(need_backward=1)
    elif case == "no_output":
        a, rgb8 = _args(out_color=None), None
    elif case == "bad_abi":
        a.abi_version = 2
    elif case == "views_times_P":
        a, views = _args(P=(2**31 - 1) // 3 + 1), 3            # 3 P > INT32_MAX
    elif case == "views_times_tiles":
        a, views = _args(W=16 * 2048, H=16 * 2048), 512          # 512 * 2048^2 = 2^31 tiles
    elif case == "missing_splat_input":
        a = _args(P=10)
        a.scales = None
    args = None if case == "args_null" else C.byref(a)
    assert L.gab200_forward_views(args, views, cams, rgb8, state, None) == -1


def test_forward_views_limits_are_exactly_the_documented_ones():
    """Just inside each limit the call passes validation: on a machine without a GPU it then fails on the device
    (GAB200_ERR_ARCH or GAB200_ERR_CUDA), never with GAB200_ERR_INVALID_ARGUMENT."""
    from gaussianavatars_b200 import _native as N

    if torch.cuda.is_available():
        pytest.skip("the calls below would run on the device")
    L = N.lib()
    st = N.FrameState()
    for a, views in ((_args(P=(2**31 - 1) // 3), 3), (_args(W=16 * 2048, H=16 * 2048), 511), (_args(), N.MAX_VIEWS)):
        assert L.gab200_forward_views(C.byref(a), views, DUMMY, DUMMY, C.byref(st), None) not in (-1, 0)


def test_camera_table_is_checked():
    from gaussianavatars_b200.rasterizer import check_camera_table

    dev = torch.device("cpu")
    ok = torch.zeros((3, 37))
    assert check_camera_table(ok, dev) is ok
    for bad in (torch.zeros(37), torch.zeros((3, 35)), torch.zeros((0, 37)), torch.zeros((3, 37), dtype=torch.float64),
                torch.zeros((37, 3)).t(), "cams"):
        with pytest.raises(ValueError, match="cameras"):
            check_camera_table(bad, dev)


def _cams(n=3, W=64, H=48):
    from gaussianavatars_b200 import synthetic as syn
    return [syn.look_at_camera(W, H, 40.0 + 3 * i, 30.0 + 2 * i) for i in range(n)]


def _raw_model(P=4, requires_grad=False):
    z = lambda *s: torch.zeros(*s, requires_grad=requires_grad)  # noqa: E731
    return SimpleNamespace(_xyz=z(P, 3), _rotation=z(P, 4), _scaling=z(P, 3), _opacity=z(P, 1),
                           _features_dc=z(P, 1, 3), _features_rest=z(P, 0, 3), active_sh_degree=0)


def test_camera_table_rows_are_the_graph_camera_blocks():
    from gaussianavatars_b200.graph import camera_block
    from gaussianavatars_b200.renderer import camera_table

    cams = _cams()
    t = camera_table(cams, torch.device("cpu"))
    assert t.shape == (3, 37) and t.dtype == torch.float32 and t.is_contiguous()
    for k, c in enumerate(cams):
        assert torch.equal(t[k], camera_block(c, fov=True))
    dev_fov = SimpleNamespace(**{n: getattr(cams[0], n) for n in ("world_view_transform", "full_proj_transform",
                                                                  "camera_center", "FoVx", "FoVy")},
                              tanfov=torch.tensor([0.25, 0.5]))
    assert torch.equal(camera_table([dev_fov], torch.device("cpu"))[0, 35:], torch.tensor([0.25, 0.5]))


def test_render_views_argument_checks():
    from gaussianavatars_b200.renderer import render_views

    bg = torch.zeros(3)
    with pytest.raises(ValueError, match="fused route"):
        render_views(_cams(), SimpleNamespace(_xyz=torch.zeros(4, 3)), None, bg)
    with pytest.raises(ValueError, match="one image size"):
        render_views(_cams(2) + _cams(1, 32, 32), _raw_model(), None, bg)
    with pytest.raises(ValueError, match="at least one camera"):
        render_views([], _raw_model(), None, bg)
    with pytest.raises(ValueError, match="width= and height="):
        render_views(torch.zeros((2, 37)), _raw_model(), None, bg)
    with pytest.raises(ValueError, match="cameras must be"):
        render_views(torch.zeros((2, 35)), _raw_model(), None, bg, width=64, height=48)


def test_rasterize_bound_views_is_forward_only():
    from gaussianavatars_b200.rasterizer import GaussianRasterizationSettings, rasterize_bound_views

    rs = GaussianRasterizationSettings(48, 64, 1.0, 1.0, torch.zeros(3), 1.0, None, None, 0, None, False, False)
    pc = _raw_model(requires_grad=True)
    args = (rs, torch.zeros((2, 37)), pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc,
            pc._features_rest)
    with pytest.raises(ValueError, match="forward only"):
        rasterize_bound_views(*args)
    with torch.no_grad(), pytest.raises(ValueError, match="display=True and/or float_image=True"):
        rasterize_bound_views(*args, display=False, float_image=False)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA tensors"):
        rasterize_bound_views(*args)


def test_graphed_render_views_per_replay_checks():
    from gaussianavatars_b200.graph import GraphedRender, camera_block

    cams = _cams()
    pc = SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3), faces=torch.zeros((2, 3)))
    for bad in (0, -1, 2.0, True, 65536):
        with pytest.raises(ValueError, match="views_per_replay"):
            GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=bad)
    with pytest.raises(ValueError, match="mesh overlay"):
        GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, mesh_opacity=0.5)
    one = GraphedRender(pc, 64, 48, torch.zeros(3))
    assert one.K == 1 and one.cam.shape == (37,) and one.camera is not None
    with pytest.raises(ValueError, match="cameras="):
        one.set_inputs(cameras=cams)

    view = GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, warm_cameras=[cams, cams[::-1]])
    assert view.K == 3 and view.cam.shape == (3, 37) and view.camera is None
    assert [w.shape for w in view._warm] == [(3, 37), (3, 37)]
    assert torch.equal(view._warm[1][0], camera_block(cams[2], fov=True))
    view.set_inputs(cameras=cams)
    for k, c in enumerate(cams):
        assert torch.equal(view.cam[k], camera_block(c, fov=True))
    table = torch.stack([camera_block(c, fov=True) for c in cams[::-1]])
    view.set_inputs(cameras=table)
    assert torch.equal(view.cam, table)
    with pytest.raises(ValueError, match="camera="):
        view.set_inputs(camera=cams[0])
    with pytest.raises(ValueError, match="3 cameras per replay"):
        view.set_inputs(cameras=cams[:2])
    with pytest.raises(ValueError, match=r"\(3, 37\)"):
        view.set_inputs(cameras=table[:, :35])
    with pytest.raises(ValueError, match="3 cameras per replay"):
        GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, warm_cameras=[cams[:1]])
    view.set_inputs(cameras=_cams(3, 80, 40))   # camera objects of another size: the frame's size follows
    assert (view.W, view.H) == (80, 40)


def test_graphed_eval_views_per_replay_checks():
    from gaussianavatars_b200.graph import GraphedEval

    cams = _cams()
    pc = SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3))
    with pytest.raises(ValueError, match="exceeds"):
        GraphedEval(pc, 64, 48, torch.zeros(3), views=2, views_per_replay=3)
    ev = GraphedEval(pc, 64, 48, torch.zeros(3), views=7, views_per_replay=3)
    assert ev.gt.shape == (3, 3, 48, 64) and ev.rows.tolist() == [0, 1, 2]
    gt = torch.arange(3 * 3 * 48 * 64, dtype=torch.int64).remainder(251).to(torch.uint8).view(3, 3, 48, 64)
    ev.set_inputs(cameras=cams, gt_u8=gt, view=4)
    assert torch.equal(ev.gt, gt) and int(ev.view) == 4 and ev.rows.tolist() == [4, 5, 6]
    with pytest.raises(IndexError):
        ev.set_inputs(view=5)                                  # rows 5 .. 7 of 7
    with pytest.raises(IndexError):
        ev.set_inputs(view=-1)
    with pytest.raises(ValueError, match="gt_u8"):
        ev.set_inputs(gt_u8=gt[0])                             # one view's ground truth
    with pytest.raises(ValueError, match="gt_u8"):
        ev.set_inputs(cameras=_cams(3, 80, 40), gt_u8=gt)      # the ground truth of the old size
    single = GraphedEval(pc, 64, 48, torch.zeros(3), views=7)
    assert single.rows is None and single.gt.shape == (3, 48, 64)
    single.set_inputs(view=6)
