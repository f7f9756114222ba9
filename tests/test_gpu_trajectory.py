"""A recorded camera path played on the device: a scheduled GraphedRender against eager render_display frame by frame,
the viewer's quantisation against its numpy expression restated in torch, and export_trajectory's PNG files, MP4 and
trajectory.json against the frames, encode_video and the reference viewer's own json (tests/golden)."""
import io
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gaussianavatars_b200 import trajectory as TR

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "trajectory_viewer.json")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def _golden():
    with open(GOLD) as f:
        return json.load(f)


def _path(g=None):
    """The fixture's 40-frame path: two keyframes, the dynamic timestep from 5 clamped at 7."""
    g = g or _golden()
    kfs = [{"rot": np.array(k["rot"], dtype=np.float64), "look_at": np.array(k["look_at"], dtype=np.float32),
            "radius": np.array(k["radius"], dtype=np.float32), "fovy": np.array(k["fovy"], dtype=np.float32),
            "interval": k["interval"]} for k in g["keyframes"]]
    return TR.CameraPath(kfs, width=g["width"], height=g["height"], dynamic=True, start_timestep=g["start_timestep"],
                         num_timesteps=g["num_timesteps"])


def _model():
    from tests.test_gpu_display import _flame_setup
    return _flame_setup(T=8)


def _cam(path, i):
    c = path.camera(i)
    return SimpleNamespace(**{k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in vars(c).items()})


def _eager(pc, path, i, bg, quantize="render"):
    from gaussianavatars_b200.renderer import render_display
    pc.select_mesh_by_timestep(path.timestep(i))
    return render_display(_cam(path, i), pc, Pipe, bg, float_image=True, quantize=quantize)


def _viewer_u8(img_chw):
    """local_viewer.py's (np.clip(rgb, 0, 1) * 255).astype(np.uint8) on a float32 (3,H,W) image, in torch."""
    return (img_chw.clamp(0, 1) * 255).to(torch.uint8).permute(1, 2, 0).contiguous()


def _render_u8(img_chw):
    return img_chw.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


def _mesh_ref(pc, path, i, base, rows, quantize):
    """The mesh over the float splat image as the viewer composites it: mesh_overlay's float composite, quantised."""
    from gaussianavatars_b200 import mesh_overlay
    pc.select_mesh_by_timestep(path.timestep(i))
    f = mesh_overlay(pc.verts, pc.faces, rows[i], base, mesh_opacity=0.5, out="float")
    return _viewer_u8(f) if quantize == "viewer" else _render_u8(f)


@pytest.mark.parametrize("mesh", [False, True])
@pytest.mark.parametrize("quantize", ["render", "viewer"])
def test_scheduled_render_equals_eager_frames(mesh, quantize):
    from gaussianavatars_b200.graph import GraphedRender
    pc = _model()
    path = _path()
    bg = torch.tensor([1.5, -0.25, 2.0 / 255.0], device=DEV)   # background pixels above 1, below 0 and on k/255
    rows = path.rows().to(DEV)
    view = GraphedRender(pc, path.W, path.H, bg, outputs="both" if not mesh else "u8", schedule=path.schedule(DEV),
                         mesh_opacity=0.5 if mesh else None, quantize=quantize)
    with pytest.raises(ValueError, match="schedule"):
        view.set_inputs(camera=_cam(path, 0), timestep=1)
    for i in range(len(path)):
        assert view.run_iterations(1) == 1
        torch.cuda.synchronize()
        shown, image = view.display.clone(), view.image.clone()
        ref = _eager(pc, path, i, bg)
        assert torch.equal(image, ref["render"]), i                    # the same float image as the eager frame
        if mesh:
            assert torch.equal(shown, _mesh_ref(pc, path, i, image, rows, quantize)), i
        elif quantize == "render":
            assert torch.equal(shown, ref["display_u8"]), i              # render.py's bytes, unchanged
        else:
            assert torch.equal(shown, _viewer_u8(image)), i
            assert torch.equal(shown, _eager(pc, path, i, bg, "viewer")["display_u8"]), i
    assert int(view.cursor.item()) == len(path)
    with pytest.raises(ValueError, match="past the schedule"):
        view.run_iterations(1)
    if not mesh:   # the frames reached values outside [0, 1]
        assert (image > 1).any() and (image < 0).any()


def test_viewer_quantisation_at_the_edges():
    """Pixels exactly on k/255 and just beside it, and far outside [0, 1]: a plain background image."""
    from gaussianavatars_b200.renderer import render_display
    pc = _model()
    path = _path()
    k = torch.arange(256, dtype=torch.float32)
    vals = torch.cat([k / 255, torch.nextafter(k / 255, torch.tensor(2.0)), torch.nextafter(k / 255, torch.tensor(-1.0)),
                      torch.tensor([-1e30, -1.0, 1.0 + 2 ** -23, 3.0, 1e30])])
    cam = _cam(path, 0)
    cam.FoVx = cam.FoVy = 0.0   # a zero field of view culls every splat: every pixel is the background
    for j in range(0, vals.numel(), 3):
        bg = torch.stack([vals[j], vals[min(j + 1, vals.numel() - 1)], vals[min(j + 2, vals.numel() - 1)]]).to(DEV)
        pc.select_mesh_by_timestep(0)
        out = render_display(cam, pc, Pipe, bg, float_image=True, quantize="viewer")
        assert torch.equal(out["display_u8"], _viewer_u8(out["render"])), bg.tolist()
        want = (np.clip(bg.cpu().numpy(), 0, 1) * 255).astype(np.uint8)
        assert (out["display_u8"].reshape(-1, 3).cpu().numpy() == want).all(), bg.tolist()


def test_split_runs_and_overflow_regrow():
    from gaussianavatars_b200.graph import GraphedRender
    pc = _model()
    path = _path()
    bg = torch.ones(3, device=DEV)
    view = GraphedRender(pc, path.W, path.H, bg, outputs="u8", schedule=path.schedule(DEV), quantize="viewer",
                         capacity=2048)   # far too small: the first replay overflows
    done = 0
    for n in (3, 10, 1, 26):
        assert view.run_iterations(n) == n
        done += n
        assert int(view.cursor.item()) == done
        torch.cuda.synchronize()
        assert torch.equal(view.display, _eager(pc, path, done - 1, bg, "viewer")["display_u8"]), done
    assert view.captures >= 2 and view.slot.capacity > 2048
    view.set_cursor(0)
    assert view.run_all() == len(path)
    torch.cuda.synchronize()
    assert torch.equal(view.display, _eager(pc, path, len(path) - 1, bg, "viewer")["display_u8"])


@pytest.mark.parametrize("mesh", [False, True])
def test_export_writes_the_viewer_files(mesh, tmp_path):
    from PIL import Image
    from gaussianavatars_b200 import encode_video
    from gaussianavatars_b200.trajectory import export_trajectory
    g = _golden()
    pc = _model()
    path = _path(g)
    bg = torch.ones(3, device=DEV)
    out = tmp_path / "export"
    video = tmp_path / "path.mp4"
    res = export_trajectory(pc, path, str(out), bg=bg, mesh_opacity=0.5 if mesh else None, video=str(video), gop=25,
                            batch=16, ref_json=g["ref_json"], capacity=None if mesh else 2048)
    assert res["frames"] == len(path) == 40
    if not mesh:
        assert res["captures"] >= 2   # the forced-small capacity overflowed and the batch was played again
    rows = path.rows().to(DEV)
    frames = []
    for i in range(len(path)):
        ref = _eager(pc, path, i, bg)
        want = _mesh_ref(pc, path, i, ref["render"], rows, "viewer") if mesh else _viewer_u8(ref["render"])
        got = np.asarray(Image.open(io.BytesIO((out / f"{i:05d}.png").read_bytes())).convert("RGB"))
        assert np.array_equal(got, want.cpu().numpy()), i
        frames.append(want)
    assert not (out / f"{len(path):05d}.png").exists()
    assert video.read_bytes() == encode_video(torch.stack(frames), fps=25, qp=20, gop=25)
    with open(out / "trajectory.json") as f:
        assert json.load(f) == g["trajectory"]   # the reference viewer's own export of this path
