"""CPU: the alpha / depth planes -- gab200_forward_depth_alpha and gab200_backward_depth_alpha (export, ctypes
signatures against the header, the argument checks that reject before any device work) and the Python refusals
(the drop-in route, K-view playback, "push" gradients) -- no compute calls (no GPU)."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from tests.test_host_multiview_train import DUMMY, _bwd, _header_params
from tests.test_host_multiview_train import _args as _views_args


def _args(**kw):
    """A single-camera frame's args (the multi-view tests' args with the camera pointers set)."""
    a = _views_args(**kw)
    a.viewmatrix = a.projmatrix = a.campos = DUMMY
    return a


def test_both_entry_points_are_exported_with_the_header_signatures():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    for s in ("gab200_forward_depth_alpha", "gab200_backward_depth_alpha"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(L, s)
    f = L.gab200_forward_depth_alpha
    assert f.restype is C.c_int64
    assert f.argtypes == [C.POINTER(N.ForwardArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                          C.POINTER(N.FrameState), C.c_void_p]
    assert _header_params("gab200_forward_depth_alpha", "int64_t") == [
        "const gab200_forward_args* args", "const float* tanfov", "float* out_alpha", "float* out_depth",
        "uint8_t* out_rgb8", "gab200_frame_state* state_out", "void* stream"]
    b = L.gab200_backward_depth_alpha
    assert b.restype is C.c_int32
    assert b.argtypes == [C.POINTER(N.BackwardArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    assert _header_params("gab200_backward_depth_alpha", "int32_t") == [
        "const gab200_backward_args* args", "const float* tanfov", "const float* dL_dalpha", "const float* dL_ddepth",
        "void* stream"]
    assert L.gab200_abi_version() == N.ABI_VERSION == 3   # new entry points, the structs are unchanged


FORWARD_CASES = ["no_plane", "args_null", "state_null", "bad_abi", "no_output", "missing_splat_input",
                 "display_only_with_backward"]


@pytest.mark.parametrize("case", FORWARD_CASES)
def test_forward_depth_alpha_rejects_bad_arguments_before_any_device_work(case):
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    st = N.FrameState()
    a, alpha, depth, rgb8, state = _args(), DUMMY, DUMMY, None, C.byref(st)
    if case == "no_plane":
        alpha = depth = None
    elif case == "state_null":
        state = None
    elif case == "bad_abi":
        a.abi_version = 2
    elif case == "no_output":
        a = _args(out_color=None)
    elif case == "missing_splat_input":
        a.scales = None
    elif case == "display_only_with_backward":   # no float image is only allowed for a forward-only display frame
        a, rgb8 = _args(out_color=None), DUMMY
        a.need_backward = 1
    args = None if case == "args_null" else C.byref(a)
    assert L.gab200_forward_depth_alpha(args, None, alpha, depth, rgb8, state, None) == -1


def _state(depth_prefix=1, views=0):
    from gaussianavatars_b200 import _native as N

    st = N.FrameState()
    st.geom_buffer = st.binning_buffer = st.image_buffer = DUMMY
    st.geom_bytes = st.binning_bytes = st.image_bytes = 2**62
    st.num_rendered = 1
    st.depth_prefix = depth_prefix
    st.reserved0 = views
    return st


BACKWARD_CASES = ["args_null", "bad_abi", "fwd_null", "state_null", "plain_state", "multiview_state", "multicast",
                  "no_dL_dout", "no_backward_forward", "no_geom_buffer"]


@pytest.mark.parametrize("case", BACKWARD_CASES)
def test_backward_depth_alpha_rejects_bad_arguments_before_any_device_work(case):
    L = __import__("gaussianavatars_b200._native", fromlist=["lib"]).lib()
    a, st = _args(), _state()
    a.need_backward = 1
    b = _bwd(a, st)
    if case == "bad_abi":
        b.abi_version = 2
    elif case == "fwd_null":
        b.fwd = None
    elif case == "state_null":
        b.state = None
    elif case == "plain_state":        # a gab200_forward / _display state: its records carry no depth
        st.depth_prefix = 0
    elif case == "multiview_state":    # a gab200_forward_views_train state
        st.reserved0 = 3
    elif case == "multicast":
        b.grads_are_multicast = 1
    elif case == "no_dL_dout":
        b.dL_dout_color = None
    elif case == "no_backward_forward":
        a.need_backward = 0
    elif case == "no_geom_buffer":
        st.geom_buffer = None
    args = None if case == "args_null" else C.byref(b)
    assert L.gab200_backward_depth_alpha(args, None, DUMMY, DUMMY, None) == -1


# ---- Python ------------------------------------------------------------------------------------------------------
def test_dropin_rasterizer_refuses_depth_alpha_and_names_the_fused_route():
    from gaussianavatars_b200.compat.diff_gaussian_rasterization import GaussianRasterizer

    r = GaussianRasterizer(raster_settings=None)
    z = torch.zeros((1, 3))
    with pytest.raises(ValueError, match="rasterize_bound"):
        r(means3D=z, means2D=z, opacities=z[:, :1], shs=z[:, None], scales=z, rotations=torch.zeros((1, 4)),
          depth_alpha=True)


def test_reference_route_render_refuses_depth_alpha():
    from gaussianavatars_b200.renderer import render

    pipe = SimpleNamespace(compute_cov3D_python=True, convert_SHs_python=False, debug=False)
    with pytest.raises(ValueError, match="fused route"):
        render(None, SimpleNamespace(), pipe, torch.zeros(3), depth_alpha=True)


def test_k_view_playback_refuses_depth_alpha():
    from gaussianavatars_b200.graph import GraphedRender

    pc = SimpleNamespace(_xyz=torch.zeros((1, 3)))
    with pytest.raises(ValueError, match="views_per_replay=1"):
        GraphedRender(pc, 16, 16, torch.zeros(3), views_per_replay=2, depth_alpha=True)


def test_push_gradients_are_refused():
    from gaussianavatars_b200.rasterizer import rasterize_bound

    sink = SimpleNamespace(symm_grad=SimpleNamespace(enabled=True, mode="push"))
    z = torch.zeros((1, 3))
    with pytest.raises(ValueError, match="push"):
        rasterize_bound(None, z, torch.zeros((1, 4)), z, torch.zeros((1, 1)), z[:, None], None, grad_sink=sink,
                        depth_alpha=True)
