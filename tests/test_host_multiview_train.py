"""CPU: the K-view training frame -- gab200_forward_views_train and gab200_backward_views (export, ctypes signatures
against the header, the argument checks that reject before any device work, the limits) and the host-side checks of
rasterize_bound_views_train and render_views_train -- no compute calls (no GPU)."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

from tests.test_host_multiview import _cams, _raw_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMMY = 0x1000   # never dereferenced: the calls below are rejected during argument validation or fail on the device


def _header_params(name, ret):
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    m = re.search(ret + r" " + name + r"\(([^)]*)\);", hdr)
    assert m, f"{name} is not declared in the header"
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_both_entry_points_are_exported_with_the_header_signatures():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    for s in ("gab200_forward_views_train", "gab200_backward_views"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(L, s)
    f = L.gab200_forward_views_train
    assert f.restype is C.c_int64
    assert f.argtypes == [C.POINTER(N.ForwardArgs), C.c_int32, C.c_void_p, C.POINTER(N.FrameState), C.c_void_p]
    assert _header_params("gab200_forward_views_train", "int64_t") == [
        "const gab200_forward_args* args", "int32_t views", "const float* cameras", "gab200_frame_state* state_out",
        "void* stream"]
    b = L.gab200_backward_views
    assert b.restype is C.c_int32
    assert b.argtypes == [C.POINTER(N.BackwardArgs), C.c_int32, C.c_void_p, C.c_void_p]
    assert _header_params("gab200_backward_views", "int32_t") == [
        "const gab200_backward_args* args", "int32_t views", "const float* cameras", "void* stream"]
    assert L.gab200_abi_version() == N.ABI_VERSION == 3   # new entry points, the structs are unchanged


def _args(P=10, W=33, H=17, out_color=DUMMY):
    from gaussianavatars_b200 import _native as N

    a = N.ForwardArgs()
    a.abi_version, a.input_mode, a.P = N.ABI_VERSION, N.INPUT_BOUND_RAW, P
    a.image_width, a.image_height = W, H
    a.bg = DUMMY
    a.out_color = out_color
    a.alloc_geom = a.alloc_binning = a.alloc_image = N.ALLOC_CALLBACK
    if P > 0:
        a.means3D = a.opacities = a.scales = a.rotations = a.sh_dc = a.radii = DUMMY
        a.sh_coeffs, a.sh_degree = 1, 0
    return a


FORWARD_CASES = ["views0", "views_negative", "views_too_many", "cameras_null", "state_null", "args_null", "no_output",
                 "bad_abi", "views_times_P", "views_times_tiles", "missing_splat_input", "activated",
                 "colors_precomp"]


@pytest.mark.parametrize("case", FORWARD_CASES)
def test_forward_views_train_rejects_bad_arguments_before_any_device_work(case):
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    st = N.FrameState()
    a, views, cams, state = _args(), 2, DUMMY, C.byref(st)
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
    elif case == "no_output":
        a = _args(out_color=None)
    elif case == "bad_abi":
        a.abi_version = 2
    elif case == "views_times_P":
        a, views = _args(P=(2**31 - 1) // 3 + 1), 3
    elif case == "views_times_tiles":
        a, views = _args(W=16 * 2048, H=16 * 2048), 512
    elif case == "missing_splat_input":
        a.scales = None
    elif case == "activated":
        a.input_mode = N.INPUT_ACTIVATED
        a.shs, a.sh_dc = DUMMY, None
    elif case == "colors_precomp":
        a.colors_precomp = DUMMY
    args = None if case == "args_null" else C.byref(a)
    assert L.gab200_forward_views_train(args, views, cams, state, None) == -1


def _state(views):
    from gaussianavatars_b200 import _native as N

    st = N.FrameState()
    st.geom_buffer = st.binning_buffer = st.image_buffer = DUMMY
    st.geom_bytes = st.binning_bytes = st.image_bytes = 2**62
    st.num_rendered = 1
    st.reserved0 = views
    return st


def _bwd(a, st):
    from gaussianavatars_b200 import _native as N

    b = N.BackwardArgs()
    b.abi_version = N.ABI_VERSION
    b.fwd, b.state = C.pointer(a), C.pointer(st)
    b.dL_dout_color = b.dL_dmeans3D = b.dL_dmeans2D = b.dL_dopacity = DUMMY
    b.dL_dsh_dc = b.dL_dscales = b.dL_drotations = DUMMY
    return b


BACKWARD_CASES = ["args_null", "bad_abi", "fwd_null", "state_null", "views0", "views_too_many", "cameras_null",
                  "single_view_state", "other_k_state", "activated", "colors_precomp", "multicast", "no_dL_dout",
                  "no_dL_dsh_dc", "no_dL_dsh_rest", "views_times_P", "not_the_forward_buffers", "no_geom_buffer"]


@pytest.mark.parametrize("case", BACKWARD_CASES)
def test_backward_views_rejects_bad_arguments_before_any_device_work(case):
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    views, cams = 2, DUMMY
    a, st = _args(), _state(2)
    b = _bwd(a, st)
    if case == "bad_abi":
        b.abi_version = 2
    elif case == "fwd_null":
        b.fwd = None
    elif case == "state_null":
        b.state = None
    elif case == "views0":
        views = 0
    elif case == "views_too_many":
        views = N.MAX_VIEWS + 1
    elif case == "cameras_null":
        cams = None
    elif case == "single_view_state":
        st.reserved0 = 0
    elif case == "other_k_state":
        st.reserved0 = 3
    elif case == "activated":
        a.input_mode = N.INPUT_ACTIVATED
        a.shs, a.sh_dc = DUMMY, None
    elif case == "colors_precomp":
        a.colors_precomp = DUMMY
    elif case == "multicast":
        b.grads_are_multicast = 1
    elif case == "no_dL_dout":
        b.dL_dout_color = None
    elif case == "no_dL_dsh_dc":
        b.dL_dsh_dc = None
    elif case == "no_dL_dsh_rest":
        a.sh_coeffs, a.sh_rest = 4, DUMMY   # dL_dsh_rest stays NULL
    elif case == "views_times_P":
        a, st, views = _args(P=(2**31 - 1) // 3 + 1), _state(3), 3
        b = _bwd(a, st)
    elif case == "not_the_forward_buffers":
        st.geom_bytes = 256
    elif case == "no_geom_buffer":
        st.geom_buffer = None
    args = None if case == "args_null" else C.byref(b)
    assert L.gab200_backward_views(args, views, cams, None) == -1


def test_single_view_backward_refuses_a_multi_view_state():
    from gaussianavatars_b200 import _native as N

    a = _args()
    a.need_backward = 1
    a.viewmatrix = a.projmatrix = a.campos = DUMMY
    b = _bwd(a, _state(2))
    assert N.lib().gab200_backward(C.byref(b), None) == -1
    assert N.lib().gab200_backward_device_fov(C.byref(b), DUMMY, None) == -1


def test_limits_are_exactly_the_documented_ones():
    """Just inside each limit the calls pass validation: without a GPU they then fail on the device, never with
    GAB200_ERR_INVALID_ARGUMENT."""
    from gaussianavatars_b200 import _native as N

    if torch.cuda.is_available():
        pytest.skip("the calls below would run on the device")
    L = N.lib()
    for a, views in ((_args(P=(2**31 - 1) // 3), 3), (_args(W=16 * 2048, H=16 * 2048), 511), (_args(), N.MAX_VIEWS)):
        st = N.FrameState()
        assert L.gab200_forward_views_train(C.byref(a), views, DUMMY, C.byref(st), None) not in (-1, 0)
        st = _state(views)
        assert L.gab200_backward_views(C.byref(_bwd(a, st)), views, DUMMY, None) not in (-1, 0)


def test_rasterize_bound_views_train_argument_checks():
    from gaussianavatars_b200.rasterizer import GaussianRasterizationSettings, rasterize_bound_views_train

    rs = GaussianRasterizationSettings(48, 64, 1.0, 1.0, torch.zeros(3), 1.0, None, None, 0, None, False, False)
    pc = _raw_model(requires_grad=True)
    args = (rs, torch.zeros((2, 37)), pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc,
            pc._features_rest)
    with pytest.raises(ValueError, match="colors_precomp"):
        rasterize_bound_views_train(*args, colors_precomp=torch.zeros((4, 3)))
    push = SimpleNamespace(symm_grad=SimpleNamespace(enabled=True, mode="push"))
    with pytest.raises(ValueError, match="'push'"):
        rasterize_bound_views_train(*args, grad_sink=push)
    for mode in ("two_shot", "plain"):   # accepted: the call goes on to the device check
        sink = SimpleNamespace(symm_grad=SimpleNamespace(enabled=True, mode=mode))
        with pytest.raises(RuntimeError, match="CUDA tensors"):
            rasterize_bound_views_train(*args, grad_sink=sink)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        rasterize_bound_views_train(*args)


def test_render_views_train_argument_checks():
    from gaussianavatars_b200.renderer import render_views_train

    bg = torch.zeros(3)
    with pytest.raises(ValueError, match="fused route"):
        render_views_train(_cams(), SimpleNamespace(_xyz=torch.zeros(4, 3)), None, bg)
    with pytest.raises(ValueError, match="one image size"):
        render_views_train(_cams(2) + _cams(1, 32, 32), _raw_model(), None, bg)
    with pytest.raises(ValueError, match="at least one camera"):
        render_views_train([], _raw_model(), None, bg)
    with pytest.raises(ValueError, match="width= and height="):
        render_views_train(torch.zeros((2, 37)), _raw_model(), None, bg)
    with pytest.raises(ValueError, match="cameras must be"):
        render_views_train(torch.zeros((2, 35)), _raw_model(), None, bg, width=64, height=48)


def _cpu_frame(monkeypatch, **kw):
    """A GraphedFrame built on the CPU: its pinned staging and loss slots become ordinary host tensors."""
    from gaussianavatars_b200.graph import GraphedFrame
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    pc = SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3))
    return GraphedFrame(pc, 64, 48, 1.0, 1.0, torch.zeros(3), **kw)


def test_graphed_frame_views_per_replay_checks(monkeypatch):
    from gaussianavatars_b200.graph import camera_block

    for bad in (0, -1, 2.0, True, 65536):
        with pytest.raises(ValueError, match="views_per_replay"):
            _cpu_frame(monkeypatch, views_per_replay=bad)
    one = _cpu_frame(monkeypatch)
    assert one.K == 1 and one.cam.shape == (35,) and one.gt.shape == (3, 48, 64)
    with pytest.raises(ValueError, match="cameras="):
        one.set_inputs(cameras=_cams())

    cams = _cams()
    fr = _cpu_frame(monkeypatch, views_per_replay=3, warm_cameras=[cams, cams[::-1]])
    assert fr.K == 3 and fr.per_camera_fov and fr.camera is None
    assert fr.cam.shape == (3, 37) and fr.gt.shape == (3, 3, 48, 64)
    assert [w.shape for w in fr._warm] == [(3, 37), (3, 37)]
    fr.set_inputs(cameras=cams)
    for k, c in enumerate(cams):
        assert torch.equal(fr.cam[k], camera_block(c, fov=True))
    table = torch.stack([camera_block(c, fov=True) for c in cams[::-1]])
    fr.set_inputs(cameras=table)
    assert torch.equal(fr.cam, table)
    gt = torch.arange(3 * 3 * 48 * 64).remainder(251).to(torch.uint8).view(3, 3, 48, 64)
    fr.set_inputs(gt_u8=gt)
    assert torch.equal(fr.gt, gt)
    with pytest.raises(ValueError, match="camera="):
        fr.set_inputs(camera=cams[0])
    with pytest.raises(ValueError, match="3 cameras per replay"):
        fr.set_inputs(cameras=cams[:2])
    with pytest.raises(ValueError, match=r"\(3, 37\)"):
        fr.set_inputs(cameras=table[:, :35])
    with pytest.raises(ValueError, match="64x48"):
        fr.set_inputs(cameras=_cams(3, 80, 40))
    with pytest.raises(ValueError, match="gt_u8"):
        fr.set_inputs(gt_u8=gt[0])
    with pytest.raises(ValueError, match="3 cameras per replay"):
        _cpu_frame(monkeypatch, views_per_replay=3, warm_cameras=[cams[:1]])

    dl = _cpu_frame(monkeypatch, views_per_replay=2, loss="dL_dimage", host_inputs=False)
    assert dl.dL_dimage.shape == (2, 3, 48, 64) and dl.gt is None
    with pytest.raises(ValueError, match="dL_dimage"):
        dl.set_inputs(dL_dimage=torch.zeros(3, 48, 64))
