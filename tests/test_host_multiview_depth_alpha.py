"""CPU: the alpha / depth planes of a K-view frame -- gab200_forward_views_depth_alpha,
gab200_forward_views_train_depth_alpha and gab200_backward_views_depth_alpha (export, ctypes signatures against the
header, the argument checks that reject before any device work) and the Python refusals -- no compute calls (no GPU)."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from tests.test_host_multiview import _raw_model
from tests.test_host_multiview_train import DUMMY, _args, _bwd, _header_params

SYMBOLS = ("gab200_forward_views_depth_alpha", "gab200_forward_views_train_depth_alpha",
           "gab200_backward_views_depth_alpha")


def test_the_three_entry_points_are_exported_with_the_header_signatures():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    for s in SYMBOLS:
        assert s in N.EXPORTED_SYMBOLS and hasattr(L, s)
    f = L.gab200_forward_views_depth_alpha
    assert f.restype is C.c_int64
    assert f.argtypes == [C.POINTER(N.ForwardArgs), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                          C.POINTER(N.FrameState), C.c_void_p]
    assert _header_params("gab200_forward_views_depth_alpha", "int64_t") == [
        "const gab200_forward_args* args", "int32_t views", "const float* cameras", "float* out_alpha",
        "float* out_depth", "uint8_t* out_rgb8", "gab200_frame_state* state_out", "void* stream"]
    t = L.gab200_forward_views_train_depth_alpha
    assert t.restype is C.c_int64
    assert t.argtypes == [C.POINTER(N.ForwardArgs), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                          C.POINTER(N.FrameState), C.c_void_p]
    assert _header_params("gab200_forward_views_train_depth_alpha", "int64_t") == [
        "const gab200_forward_args* args", "int32_t views", "const float* cameras", "float* out_alpha",
        "float* out_depth", "gab200_frame_state* state_out", "void* stream"]
    b = L.gab200_backward_views_depth_alpha
    assert b.restype is C.c_int32
    assert b.argtypes == [C.POINTER(N.BackwardArgs), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    assert _header_params("gab200_backward_views_depth_alpha", "int32_t") == [
        "const gab200_backward_args* args", "int32_t views", "const float* cameras", "const float* dL_dalpha",
        "const float* dL_ddepth", "void* stream"]
    assert L.gab200_abi_version() == N.ABI_VERSION == 3   # new entry points, the structs are unchanged


FORWARD_CASES = ["no_plane", "need_backward", "views0", "views_too_many", "cameras_null", "state_null", "args_null",
                 "no_output", "bad_abi", "views_times_P", "views_times_tiles", "missing_splat_input"]


@pytest.mark.parametrize("case", FORWARD_CASES)
def test_forward_views_depth_alpha_rejects_bad_arguments_before_any_device_work(case):
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    st = N.FrameState()
    a, views, cams, alpha, depth, rgb8, state = _args(), 2, DUMMY, DUMMY, DUMMY, None, C.byref(st)
    if case == "no_plane":
        alpha = depth = None
    elif case == "need_backward":           # the K-view forward is forward only: the training form has its own call
        a.need_backward = 1
    elif case == "views0":
        views = 0
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
    args = None if case == "args_null" else C.byref(a)
    assert L.gab200_forward_views_depth_alpha(args, views, cams, alpha, depth, rgb8, state, None) == -1


TRAIN_CASES = ["no_plane", "views0", "views_too_many", "cameras_null", "state_null", "args_null", "no_output",
               "bad_abi", "views_times_P", "views_times_tiles", "missing_splat_input", "activated", "colors_precomp"]


@pytest.mark.parametrize("case", TRAIN_CASES)
def test_forward_views_train_depth_alpha_rejects_bad_arguments_before_any_device_work(case):
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    st = N.FrameState()
    a, views, cams, alpha, depth, state = _args(), 2, DUMMY, DUMMY, DUMMY, C.byref(st)
    if case == "no_plane":
        alpha = depth = None
    elif case == "views0":
        views = 0
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
    assert L.gab200_forward_views_train_depth_alpha(args, views, cams, alpha, depth, state, None) == -1


def _state(views, depth_prefix=1):
    from gaussianavatars_b200 import _native as N

    st = N.FrameState()
    st.geom_buffer = st.binning_buffer = st.image_buffer = DUMMY
    st.geom_bytes = st.binning_bytes = st.image_bytes = 2**62
    st.num_rendered = 1
    st.reserved0 = views
    st.depth_prefix = depth_prefix
    return st


BACKWARD_CASES = ["args_null", "bad_abi", "fwd_null", "state_null", "views0", "views_too_many", "cameras_null",
                  "plain_k_view_state", "single_view_state", "other_k_state", "activated", "colors_precomp",
                  "multicast", "no_dL_dout", "no_dL_dsh_dc", "no_dL_dsh_rest", "views_times_P",
                  "not_the_forward_buffers", "no_geom_buffer"]


@pytest.mark.parametrize("case", BACKWARD_CASES)
def test_backward_views_depth_alpha_rejects_bad_arguments_before_any_device_work(case):
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
    elif case == "plain_k_view_state":    # a gab200_forward_views_train state: its records carry no depth
        st.depth_prefix = 0
    elif case == "single_view_state":     # a gab200_forward_depth_alpha state
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
    assert L.gab200_backward_views_depth_alpha(args, views, cams, DUMMY, DUMMY, None) == -1


def test_single_view_depth_alpha_backward_refuses_a_k_view_depth_alpha_state():
    from gaussianavatars_b200 import _native as N

    a = _args()
    a.need_backward = 1
    a.viewmatrix = a.projmatrix = a.campos = DUMMY
    b = _bwd(a, _state(2))
    assert N.lib().gab200_backward_depth_alpha(C.byref(b), None, DUMMY, DUMMY, None) == -1


def test_limits_are_those_of_the_k_view_entry_points():
    """Just inside each limit the calls pass validation: without a GPU they then fail on the device, never with
    GAB200_ERR_INVALID_ARGUMENT."""
    from gaussianavatars_b200 import _native as N

    if torch.cuda.is_available():
        pytest.skip("the calls below would run on the device")
    L = N.lib()
    for a, views in ((_args(P=(2**31 - 1) // 3), 3), (_args(W=16 * 2048, H=16 * 2048), 511), (_args(), N.MAX_VIEWS)):
        st = N.FrameState()
        assert L.gab200_forward_views_depth_alpha(C.byref(a), views, DUMMY, DUMMY, None, None, C.byref(st),
                                                  None) not in (-1, 0)
        st = N.FrameState()
        assert L.gab200_forward_views_train_depth_alpha(C.byref(a), views, DUMMY, None, DUMMY, C.byref(st),
                                                        None) not in (-1, 0)
        st = _state(views)
        assert L.gab200_backward_views_depth_alpha(C.byref(_bwd(a, st)), views, DUMMY, None, None,
                                                   None) not in (-1, 0)


# ---- Python ------------------------------------------------------------------------------------------------------
def test_rasterize_bound_views_train_with_planes_argument_checks():
    from gaussianavatars_b200.rasterizer import GaussianRasterizationSettings, rasterize_bound_views_train

    rs = GaussianRasterizationSettings(48, 64, 1.0, 1.0, torch.zeros(3), 1.0, None, None, 0, None, False, False)
    pc = _raw_model(requires_grad=True)
    args = (rs, torch.zeros((2, 37)), pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc,
            pc._features_rest)
    with pytest.raises(ValueError, match="colors_precomp"):
        rasterize_bound_views_train(*args, colors_precomp=torch.zeros((4, 3)), depth_alpha=True)
    push = SimpleNamespace(symm_grad=SimpleNamespace(enabled=True, mode="push"))
    with pytest.raises(ValueError, match="'push'"):
        rasterize_bound_views_train(*args, grad_sink=push, depth_alpha=True)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        rasterize_bound_views_train(*args, depth_alpha=True)


def test_rasterize_bound_views_with_planes_argument_checks():
    from gaussianavatars_b200.rasterizer import GaussianRasterizationSettings, rasterize_bound_views

    rs = GaussianRasterizationSettings(48, 64, 1.0, 1.0, torch.zeros(3), 1.0, None, None, 0, None, False, False)
    pc = _raw_model(requires_grad=True)
    args = (rs, torch.zeros((2, 37)), pc._xyz, pc._rotation, pc._scaling, pc._opacity, pc._features_dc,
            pc._features_rest)
    with pytest.raises(ValueError, match="forward only"):
        rasterize_bound_views(*args, depth_alpha=True)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA tensors"):
        rasterize_bound_views(*args, depth_alpha=True)


def test_render_views_with_planes_need_the_fused_route():
    from gaussianavatars_b200.renderer import render_views, render_views_train

    bg = torch.zeros(3)
    no_raw = SimpleNamespace(_xyz=torch.zeros(4, 3))
    with pytest.raises(ValueError, match="fused route"):
        render_views_train(torch.zeros((2, 37)), no_raw, None, bg, width=64, height=48, depth_alpha=True)
    with pytest.raises(ValueError, match="fused route"):
        render_views(torch.zeros((2, 37)), no_raw, None, bg, width=64, height=48, depth_alpha=True)
