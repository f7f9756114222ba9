"""-m gpu: the display image written by the forward blend (gab200_forward_display, rasterize_bound(rgb8=),
render_display) and the forward-only playback graph (GraphedRender).

Every comparison is bit for bit: the display image against torch's quantisation of the float image
(mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(uint8), render.py), the float image against the existing
entry point, and a replay against the eager render_display of the same inputs."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import helpers as h
from tests.test_gpu_camera_fov import _dev_tanfov, _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


@pytest.fixture(autouse=True)
def culled_binning():
    """The library's default binning policy, whatever an earlier test left set (the policy is process-wide); the
    display epilogue does not depend on it, but the instance counts the capacities here are sized for do."""
    import gaussianavatars_b200.rasterizer as R
    prev = R._EXACT_BINNING
    R.set_exact_binning(False)
    yield
    R.set_exact_binning(prev)


def _quant(img):
    """render.py's conversion of the float image, on the device."""
    return img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


# ---- quantisation -------------------------------------------------------------------------------------------------
def _bg_values():
    f = np.float32
    vals = []
    for k in range(256):
        vals.append(f(k) / f(255))
        mid = (f(k) + f(0.5)) / f(255)
        vals += [mid, np.nextafter(mid, f(-1)), np.nextafter(mid, f(2))]
    vals += [-1.0, -1e-3, -0.0, -1e-30, 1.0 + 1e-6, 1.002, 2.0, 1e6, -1e6, np.inf, -np.inf]
    v = np.array(vals, np.float32)
    return np.concatenate([v, np.zeros((-len(v)) % 3, np.float32)]).reshape(-1, 3)


@pytest.mark.parametrize("W,H", [(64, 32), (37, 19)])   # whole-word rows; byte rows (W % 4 != 0)
def test_empty_scene_quantises_every_background_exactly(W, H):
    import gaussianavatars_b200.rasterizer as R
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import synthetic as syn
    bgs = _bg_values()
    assert bgs.size >= 512
    cam = syn.look_at_camera(W, H, 40.0, 30.0)
    for bg in bgs:
        sc = dict(cam=cam, W=W, H=H, bg=torch.from_numpy(bg.copy()), sh_degree=0)
        rs = h.cuda_settings(sc, DEV, debug=False)
        a = N.ForwardArgs()
        keep = R._fill_common(a, rs, DEV, 0, False)
        a.input_mode = N.INPUT_BOUND_RAW
        rgb8 = torch.full((H, W, 3), 7, dtype=torch.uint8, device=DEV)
        img, *_ = R._run_forward(a, DEV, False, R.FrameHints(), None, rgb8, True)
        both = rgb8.clone()
        rgb8.fill_(7)
        none, *_ = R._run_forward(a, DEV, False, R.FrameHints(), None, rgb8, False)
        assert none is None
        want = _quant(torch.from_numpy(bg.copy()).to(DEV).view(3, 1, 1).expand(3, H, W).contiguous())
        assert torch.equal(img, torch.from_numpy(bg.copy()).to(DEV).view(3, 1, 1).expand(3, H, W)), bg
        assert torch.equal(both, _quant(img)), f"background {bg.tolist()}"
        assert torch.equal(both, want) and torch.equal(rgb8, both), f"background {bg.tolist()}"
        del keep


# ---- full scenes, every sync mode ----------------------------------------------------------------------------------
class _Sync:
    """Runs a call under one of the three sync modes: LATE with a capacity far too small (the re-enqueue path runs),
    NONE with a fixed `capacity` that must fit the frame (its sticky overflow flag must stay clear)."""

    def __init__(self, mode, key, capacity=0):
        self.mode, self.key, self.capacity = mode, key, capacity

    def __call__(self, fn):
        import gaussianavatars_b200.rasterizer as R
        hints = R.FrameHints()
        R.set_sync_policy("exact" if self.mode == "exact" else "late")
        slot = None
        try:
            if self.mode == "late":
                hints.set_capacity(self.key, 1024)
                hints.set_depth(self.key, (0, 0))
            if self.mode == "none":
                slot = R._capture_slot = R.CaptureSlot(DEV, self.capacity)
            out = fn(hints)
        finally:
            R._capture_slot = None
            R.set_sync_policy("late")
        if self.mode == "late":
            assert R.last_frame_info()["attempts"] == 2 and R.last_frame_info()["sync_mode"] == 1
        if slot is not None:
            torch.cuda.synchronize()
            assert int(slot.flag.item()) == 0, \
                f"the NONE-mode frame overflowed its capacity: counters {slot.counters.tolist()} {R.last_frame_info()}"
        return out


def _display_run(sc, cam, sync, mode):
    """No-grad fused forward with the device field of view; mode None (gab200_forward_device_fov), "both", "u8"."""
    from gaussianavatars_b200.rasterizer import face_frame, rasterize_bound
    p = sc["params"]
    leaves = [p[k].to(DEV).contiguous() for k in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc",
                                                   "_features_rest")]
    fc, fR, fs = face_frame(sc["verts"].to(DEV), sc["faces"].to(DEV))
    rs = h.cuda_settings(dict(cam=cam, W=sc["W"], H=sc["H"], bg=sc["bg"], sh_degree=3), DEV, debug=False)
    rgb8 = torch.empty((sc["H"], sc["W"], 3), dtype=torch.uint8, device=DEV) if mode else None
    tanfov = _dev_tanfov(cam)

    def go(hints):
        with torch.no_grad():
            return rasterize_bound(rs, *leaves, binding=p["binding"].to(DEV), face_center=fc, face_orien_mat=fR,
                                   face_scaling=fs, grad_sink=SimpleNamespace(_gab200_hints=hints), tanfov=tanfov,
                                   rgb8=rgb8, float_image=mode != "u8")
    img, radii = sync(go)
    torch.cuda.synchronize()
    return img, radii, rgb8


@pytest.mark.parametrize("P,W,H", [(100_000, 1920, 1080), (150_000, 550, 802), (60_000, 333, 250),
                                   (60_000, 500, 301)])
def test_display_image_in_every_sync_mode(P, W, H):
    sc = h.avatar_scene(P=P, W=W, H=H, seed=4)
    sc["bg"] = torch.tensor([0.3, 0.55, 1.0])
    cam = sc["cam"]
    key = (DEV, W, H, P)
    ref_img, ref_radii, _ = _display_run(sc, cam, _Sync("exact", key), None)
    import gaussianavatars_b200.rasterizer as R
    cap = 2 * R.last_frame_info()["num_rendered"] + 4096   # the NONE-mode frames' capacity: room for this frame
    assert int((ref_radii > 0).sum()) > 1000, "scene renders nothing"
    want = _quant(ref_img)
    assert len(torch.unique(want)) > 100
    for sync in ("exact", "late", "none"):
        img, radii, u8 = _display_run(sc, cam, _Sync(sync, key, cap), "both")
        assert torch.equal(img, ref_img), f"{sync}: float image differs from gab200_forward_device_fov"
        assert torch.equal(radii, ref_radii), sync
        assert torch.equal(u8, _quant(img)), f"{sync}: display image differs from the torch quantisation"
        none, radii, u8only = _display_run(sc, cam, _Sync(sync, key, cap), "u8")
        assert none is None and torch.equal(u8only, want), f"{sync}: u8-only display image differs"


def test_render_display_matches_render():
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render, render_display
    sc = h.avatar_scene(P=30_000, W=480, H=352, seed=2)
    pc = MeshBoundGaussians(sc["params"], 3, sc["verts"], sc["faces"], pose_fn=syn.pose_mesh, device=DEV)
    pc.update_mesh_properties(sc["verts"].to(DEV))
    cam = sc["cam"].to(DEV)
    bg = torch.tensor([0.0, 0.5, 1.0], device=DEV)
    with torch.no_grad():
        ref = render(cam, pc, Pipe, bg)
    out = render_display(cam, pc, Pipe, bg, float_image=True)
    assert torch.equal(out["render"], ref["render"]) and torch.equal(out["radii"], ref["radii"])
    assert torch.equal(out["visibility_filter"], ref["visibility_filter"])
    assert torch.equal(out["display_u8"], _quant(ref["render"]))
    only = render_display(cam, pc, Pipe, bg)
    assert only["render"] is None and torch.equal(only["display_u8"], out["display_u8"])


# ---- GraphedRender against eager render_display ---------------------------------------------------------------------
def _flame_setup(T=8):
    from tests.test_gpu_flame import _flame_model, _full_size, _lbs
    a, fp = _full_size(T=T, seed=2)
    return _flame_model(a, fp, _lbs(a))


W_IMG, H_IMG = 400, 304


def _eager(pc, cam, t, bg, scaling_modifier=1.0):
    from gaussianavatars_b200.renderer import render_display
    pc.select_mesh_by_timestep(t)
    out = render_display(cam.to(DEV), pc, Pipe, bg.to(DEV), scaling_modifier, float_image=True)
    torch.cuda.synchronize()
    return out


def _same(view, ref, what):
    torch.cuda.synchronize()
    assert torch.equal(view.image, ref["render"]), f"{what}: float image differs"
    assert torch.equal(view.display, ref["display_u8"]), f"{what}: display image differs"
    assert torch.equal(view.radii, ref["radii"]), f"{what}: radii differ"


def test_graphed_render_follows_timesteps_cameras_background_and_edits():
    from gaussianavatars_b200.graph import GraphedRender
    pc = _flame_setup()
    cams = _rig(W_IMG, H_IMG)
    bg = torch.tensor([1.0, 1.0, 1.0])
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", warm_cameras=cams, warm_timesteps=range(8))
    view.set_inputs(camera=cams[0], timestep=0)
    for t in list(range(8)) + list(range(6, -1, -1)):
        view.set_inputs(timestep=t)
        view.run(check=True)
        _same(view, _eager(pc, cams[0], t, bg), f"timestep {t}")
    assert view.captures == 1
    for i, cam in enumerate(cams):
        view.set_inputs(camera=cam, timestep=i % 8)
        view.run(check=True)
        _same(view, _eager(pc, cam, i % 8, bg), f"camera {i}")
    assert view.captures == 1

    bg2 = torch.tensor([0.1, 0.45, 0.8])
    view.set_inputs(camera=cams[3], timestep=2, bg=bg2.to(DEV))
    view.run(check=True)
    _same(view, _eager(pc, cams[3], 2, bg2), "new background")
    assert view.captures == 1

    before = view.display.clone()
    with torch.no_grad():
        pc.flame_param["jaw_pose"][2] += torch.tensor([0.25, 0.0, 0.0], device=DEV)
    view.run(check=True)
    torch.cuda.synchronize()
    assert not torch.equal(view.display, before), "the jaw edit changed nothing"
    _same(view, _eager(pc, cams[3], 2, bg2), "jaw-pose edit")
    assert view.captures == 1

    view.scaling_modifier = 0.8
    view.run(check=True)
    _same(view, _eager(pc, cams[3], 2, bg2, 0.8), "scaling_modifier")
    assert view.captures == 2
    pc.active_sh_degree = 1
    view.run(check=True)
    _same(view, _eager(pc, cams[3], 2, bg2, 0.8), "active_sh_degree")
    assert view.captures == 3
    assert not view.overflowed()


def test_graphed_render_capacity_guard():
    from gaussianavatars_b200.graph import GraphedRender
    pc = _flame_setup(T=6)
    cam = _rig(W_IMG, H_IMG, n=4)[1]
    bg = torch.ones(3)
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", capacity=2000)
    view.set_inputs(camera=cam, timestep=1)
    view.run(check=False)
    assert view.overflowed()
    view.run(check=True)
    assert not view.overflowed() and view.captures == 2
    _same(view, _eager(pc, cam, 1, bg), "after regrow")


def test_graphed_render_owns_its_scratch():
    """A larger eager no_grad frame grows (replaces) the pooled inference scratch; the graph must not care."""
    from gaussianavatars_b200.graph import GraphedRender
    from gaussianavatars_b200.renderer import render_display
    pc = _flame_setup(T=6)
    cam = _rig(W_IMG, H_IMG, n=4)[2]
    bg = torch.ones(3)
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", capacity=3_000_000)
    view.set_inputs(camera=cam, timestep=3)
    view.run(check=True)
    torch.cuda.synchronize()
    first = (view.image.clone(), view.display.clone(), view.radii.clone())
    big = _rig(1920, 1080, n=4)[2]
    pc.select_mesh_by_timestep(0)
    render_display(big.to(DEV), pc, Pipe, bg.to(DEV), float_image=True)          # the pool grows
    render_display(cam.to(DEV), pc, Pipe, torch.zeros(3, device=DEV), float_image=True)
    view.run(check=True)
    torch.cuda.synchronize()
    assert torch.equal(view.image, first[0]) and torch.equal(view.display, first[1])
    assert torch.equal(view.radii, first[2]) and view.captures == 1


def test_graphed_render_host_ring():
    from gaussianavatars_b200.graph import GraphedRender
    pc = _flame_setup(T=8)
    cams = _rig(W_IMG, H_IMG, n=8)
    k = 3
    view = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", host_slots=k, warm_cameras=cams,
                         warm_timesteps=range(8))
    frames = []
    for i in range(32):
        view.set_inputs(camera=cams[i % 8], timestep=(3 * i) % 8)
        view.run()
        assert view.image is None
        frames.append(view.display.clone())   # stream-ordered behind replay i, before replay i + 1
        if i >= 1:   # the consumer one replay behind
            assert torch.equal(view.host_frame(i - 1), frames[i - 1].cpu()), f"slot of replay {i - 1}"
        for j in range(max(0, i - k + 1), i + 1):   # the last k replays are all still in the ring
            assert torch.equal(view.host_frame(j), frames[j].cpu()), f"replay {j} overwritten at replay {i}"
        if i >= k:
            with pytest.raises(IndexError):
                view.host_frame(i - k)
    assert len({bytes(f.cpu().numpy().tobytes()[:4096]) for f in frames[:8]}) > 1
    assert view.captures == 1 and not view.overflowed()


def test_graphed_render_and_training_frame_interleave():
    """A training preview: a GraphedFrame and a GraphedRender on the same model, replayed alternately."""
    from gaussianavatars_b200.graph import GraphedFrame, GraphedRender, camera_block
    from gaussianavatars_b200.renderer import render
    pc = _flame_setup(T=6)
    cams = _rig(W_IMG, H_IMG, n=6)
    bg = torch.ones(3)
    gt = torch.randint(0, 256, (3, H_IMG, W_IMG), generator=torch.Generator().manual_seed(7),
                       dtype=torch.uint8).to(DEV)
    blocks = [camera_block(c, fov=True).to(DEV) for c in cams]
    fr = GraphedFrame(pc, W_IMG, H_IMG, cams[0].FoVx, cams[0].FoVy, bg, loss="l1_u8", per_camera_fov=True,
                      warm_cameras=blocks)
    fr.set_inputs(camera=blocks[0], gt_u8=gt, timestep=0)
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", warm_cameras=cams, warm_timesteps=range(6))
    for i in range(6):
        fr.set_inputs(camera=cams[i])   # the training frame stays at timestep 0, the preview walks the sequence
        fr.run(check=True)
        view.set_inputs(camera=cams[5 - i], timestep=5 - i)
        view.run(check=True)
        torch.cuda.synchronize()
        pc.select_mesh_by_timestep(0)
        ref = render(cams[i].to(DEV), pc, Pipe, bg.to(DEV))["render"].detach()
        torch.cuda.synchronize()
        assert torch.equal(fr.image, ref), f"step {i}: training replay differs from eager render()"
        assert math.isfinite(float(fr.loss))
        _same(view, _eager(pc, cams[5 - i], 5 - i, bg), f"step {i}: playback replay")
    assert fr.captures == 1 and view.captures == 1
