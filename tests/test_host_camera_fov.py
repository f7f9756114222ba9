"""CPU: the per-camera field of view read from device memory -- the new entry points, the 37-float camera block and
the host-side argument checks of GraphedFrame(per_camera_fov=True) and of render() -- no compute calls (no GPU)."""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def test_device_fov_entry_points_are_exported_and_reject_bad_arguments():
    from gaussianavatars_b200 import _native as N

    lib = N.lib()
    for s in ("gab200_forward_device_fov", "gab200_backward_device_fov"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(lib, s)
    assert lib.gab200_abi_version() == N.ABI_VERSION == 3
    st = N.FrameState()
    assert lib.gab200_forward_device_fov(None, None, C.byref(st), None) == -1
    a = N.ForwardArgs()   # abi_version 0
    assert lib.gab200_forward_device_fov(C.byref(a), None, C.byref(st), None) == -1
    assert lib.gab200_backward_device_fov(None, None, None) == -1
    b = N.BackwardArgs()
    b.abi_version = N.ABI_VERSION
    assert lib.gab200_backward_device_fov(C.byref(b), None, None) == -1   # no forward args / state


def _cams():
    from gaussianavatars_b200 import synthetic as syn
    return [syn.orbit_camera(550, 802, azimuth_deg=30.0),
            syn.look_at_camera(64, 48, 37.3, 28.9, w2c=np.diag([1.0, -1.0, -1.0, 1.0]) @ np.eye(4)),
            syn.look_at_camera(33, 17, 90.0, 90.0)]


def test_camera_block_with_fov_appends_the_rounded_tangents():
    from gaussianavatars_b200.graph import camera_block

    for cam in _cams():
        b35, b37 = camera_block(cam), camera_block(cam, fov=True)
        assert b35.shape == (35,) and b37.shape == (37,) and b37.dtype == torch.float32
        assert torch.equal(b37[:35], b35)
        # exactly what render()'s settings hand to the kernels: tan in double, rounded to float32 once
        assert float(b37[35]) == C.c_float(math.tan(cam.FoVx * 0.5)).value == float(np.float32(math.tan(cam.FoVx / 2)))
        assert float(b37[36]) == C.c_float(math.tan(cam.FoVy * 0.5)).value


def _cpu_model():
    return SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3))


def test_graphed_frame_per_camera_fov_argument_checks(monkeypatch):
    from gaussianavatars_b200.graph import GraphedFrame, camera_block, tanfov_floats

    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)   # the frame's loss slot; no driver here

    cam = _cams()[1]
    fovx, fovy = 0.7, 0.5
    fr = GraphedFrame(_cpu_model(), 64, 48, fovx, fovy, torch.zeros(3), per_camera_fov=True)
    assert fr.cam.shape == (37,)
    assert torch.equal(fr.cam[35:], tanfov_floats(fovx, fovy))          # fovx / fovy seed the initial block
    assert fr.camera.tanfov.data_ptr() == fr.cam[35:].data_ptr()          # the kernels read the static block
    fr.set_inputs(camera=cam)                                             # a camera object fills all 37 floats
    assert torch.equal(fr.cam, camera_block(cam, fov=True))
    with pytest.raises(ValueError, match="37"):
        fr.set_inputs(camera=camera_block(cam))                           # 35 floats: no field of view
    with pytest.raises(ValueError, match="37"):
        GraphedFrame(_cpu_model(), 64, 48, fovx, fovy, torch.zeros(3), per_camera_fov=True,
                     warm_cameras=[camera_block(cam)])
    fr2 = GraphedFrame(_cpu_model(), 64, 48, fovx, fovy, torch.zeros(3), per_camera_fov=True, warm_cameras=[cam])
    assert fr2._warm[0].shape == (37,)

    # default mode: unchanged 35-float block, no device field of view
    fr0 = GraphedFrame(_cpu_model(), 64, 48, fovx, fovy, torch.zeros(3))
    assert fr0.cam.shape == (35,) and fr0.camera.tanfov is None
    fr0.set_inputs(camera=cam)
    assert torch.equal(fr0.cam, camera_block(cam))

    # a prefetching pair must agree on the mode
    a, b = SimpleNamespace(host_inputs=True, per_camera_fov=True), SimpleNamespace(host_inputs=True, per_camera_fov=False)
    with pytest.raises(ValueError, match="per_camera_fov"):
        GraphedFrame.prefetch_for(a, b)


def test_reference_route_refuses_a_device_field_of_view():
    from gaussianavatars_b200.renderer import render

    cam = _cams()[2]
    cam.tanfov = torch.tensor([1.0, 1.0])
    pc = SimpleNamespace(get_xyz=torch.zeros(4, 3))    # no raw parameters: the reference route
    with pytest.raises(ValueError, match="tanfov"):
        render(cam, pc, SimpleNamespace(), torch.zeros(3))
