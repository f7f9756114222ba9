"""CPU: the playback surface -- the gab200_forward_display entry point (export, ctypes signature, argument checks that
reject before any device work), the display-image argument check of the fused route and the host-side checks of
GraphedRender -- no compute calls (no GPU)."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMMY = 0x1000   # never dereferenced: every call below is rejected during argument validation


def test_forward_display_is_exported_with_the_header_signature():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    assert "gab200_forward_display" in N.EXPORTED_SYMBOLS and hasattr(L, "gab200_forward_display")
    assert L.gab200_abi_version() == N.ABI_VERSION == 3
    f = L.gab200_forward_display
    assert f.restype is C.c_int64
    assert f.argtypes == [C.POINTER(N.ForwardArgs), C.c_void_p, C.c_void_p, C.POINTER(N.FrameState), C.c_void_p]
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    m = re.search(r"int64_t gab200_forward_display\(([^)]*)\);", hdr)
    assert m, "gab200_forward_display is not declared in the header"
    params = [p.strip() for p in m.group(1).split(",")]
    assert params == ["const gab200_forward_args* args", "const float* tanfov", "uint8_t* out_rgb8",
                      "gab200_frame_state* state_out", "void* stream"]


def _args(need_backward=0, out_color=DUMMY):
    from gaussianavatars_b200 import _native as N

    a = N.ForwardArgs()
    a.abi_version, a.input_mode, a.P = N.ABI_VERSION, N.INPUT_BOUND_RAW, 0
    a.image_width, a.image_height = 33, 17
    a.need_backward = need_backward
    a.bg = a.viewmatrix = a.projmatrix = a.campos = DUMMY
    a.out_color = out_color
    a.alloc_geom = a.alloc_binning = a.alloc_image = N.ALLOC_CALLBACK
    return a


@pytest.mark.parametrize("need_backward, out_color, out_rgb8", [
    (1, None, DUMMY),    # no float image, but a backward needs it
    (0, None, None),     # no output at all
    (1, None, None),
])
def test_forward_display_rejects_missing_outputs(need_backward, out_color, out_rgb8):
    from gaussianavatars_b200 import _native as N

    st = N.FrameState()
    a = _args(need_backward, out_color)
    assert N.lib().gab200_forward_display(C.byref(a), None, out_rgb8, C.byref(st), None) == -1


def test_forward_display_rejects_null_args_and_state_and_keeps_the_old_entry_points_strict():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    st = N.FrameState()
    assert L.gab200_forward_display(None, None, DUMMY, C.byref(st), None) == -1
    assert L.gab200_forward_display(C.byref(_args(0, None)), None, DUMMY, None, None) == -1
    bad = _args(0, None)
    bad.abi_version = 2
    assert L.gab200_forward_display(C.byref(bad), None, DUMMY, C.byref(st), None) == -1
    # a NULL float image is only ever allowed through the display entry point
    assert L.gab200_forward(C.byref(_args(0, None)), C.byref(st), None) == -1
    assert L.gab200_forward_device_fov(C.byref(_args(0, None)), None, C.byref(st), None) == -1


def test_rgb8_destination_is_checked():
    from gaussianavatars_b200.rasterizer import check_rgb8

    rs = SimpleNamespace(image_height=17, image_width=33)
    dev = torch.device("cpu")
    assert check_rgb8(None, rs, dev) is None
    ok = torch.empty((17, 33, 3), dtype=torch.uint8)
    assert check_rgb8(ok, rs, dev) is ok
    for bad in (torch.empty((3, 17, 33), dtype=torch.uint8), torch.empty((17, 33, 3), dtype=torch.float32),
                torch.empty((17, 66, 3), dtype=torch.uint8)[:, ::2]):
        with pytest.raises(ValueError, match="rgb8"):
            check_rgb8(bad, rs, dev)


def _cams():
    from gaussianavatars_b200 import synthetic as syn
    return [syn.orbit_camera(64, 48, azimuth_deg=30.0), syn.look_at_camera(64, 48, 37.3, 28.9)]


def test_graphed_render_argument_checks():
    from gaussianavatars_b200.graph import GraphedRender, camera_block

    cam = _cams()[0]
    pc = SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3))
    view = GraphedRender(pc, 64, 48, torch.zeros(3))
    assert view.cam.shape == (37,) and view.camera.tanfov.data_ptr() == view.cam[35:].data_ptr()
    view.set_inputs(camera=cam, verts=torch.ones(5, 3), bg=torch.tensor([0.1, 0.2, 0.3]))
    assert torch.equal(view.cam, camera_block(cam, fov=True))
    assert torch.equal(view.verts, torch.ones(5, 3)) and torch.equal(view.bg, torch.tensor([0.1, 0.2, 0.3]))
    with pytest.raises(ValueError, match="37"):
        view.set_inputs(camera=camera_block(cam))                        # 35 floats: no field of view
    with pytest.raises(ValueError, match="37"):
        GraphedRender(pc, 64, 48, torch.zeros(3), warm_cameras=[camera_block(cam)])
    with pytest.raises(ValueError, match="FLAME"):
        view.set_inputs(timestep=0)                                      # no FLAME head
    with pytest.raises(ValueError, match="outputs"):
        GraphedRender(pc, 64, 48, torch.zeros(3), outputs="rgba")
    with pytest.raises(ValueError, match="host_slots"):
        GraphedRender(pc, 64, 48, torch.zeros(3), outputs="float", host_slots=2)
    assert GraphedRender(pc, 64, 48, torch.zeros(3), warm_cameras=_cams())._warm[1].shape == (37,)

    head = SimpleNamespace(_xyz=torch.zeros(4, 3), flame=object(), flame_param={"expr": torch.zeros(6, 10)})
    fv = GraphedRender(head, 64, 48, torch.zeros(3))
    with pytest.raises(ValueError, match="timestep"):
        fv.set_inputs(verts=torch.zeros(5, 3))                           # the head is posed inside the graph
    with pytest.raises(IndexError):
        fv.set_inputs(timestep=6)
    fv.set_inputs(timestep=5)
    assert int(fv.timestep) == 5
