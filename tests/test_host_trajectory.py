"""CameraPath against the reference local viewer itself: its timeline (update_record_timeline), its camera
(apply_state_dict, OrbitCamera, prepare_camera) and its trajectory.json (export_trajectory), run on the CPU with the
GUI stubbed.  Skipped where the reference is not mounted."""
import json
import sys
import types
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gaussianavatars_b200 import trajectory as TR
from gaussianavatars_b200.graph import camera_block
from tests import ref_import

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="the reference is not mounted")


def _reference():
    ref_import.prepare()
    sys.modules.setdefault("tyro", types.ModuleType("tyro"))
    import local_viewer
    from utils import viewer_utils
    return local_viewer, viewer_utils


def _viewer(keyframes, W, H, cycles, convention, tmp_path, T=1, timestep=0, dynamic=False, ref_json=None):
    """A LocalViewer without its GUI: dearpygui's values live in a dict, the render loop is not running."""
    lv, vu = _reference()
    dpg = sys.modules["dearpygui.dearpygui"]
    values = {"_input_cycles": cycles, "_checkbox_dynamic_record": dynamic, "_slider_record_timestep": 0,
              "_slider_timestep": timestep}
    dpg.get_value = lambda tag: values[tag]
    dpg.set_value = lambda tag, v: values.__setitem__(tag, v)
    dpg.configure_item = lambda *a, **k: None
    dpg.destroy_context = lambda: None
    v = lv.LocalViewer.__new__(lv.LocalViewer)
    v.cfg = SimpleNamespace(save_folder=tmp_path / "viewer", ref_json=ref_json, fps=25, keyframe_interval=1)
    v.keyframes, v.all_frames, v.num_record_timeline = list(keyframes), {}, 0
    v.cam = vu.OrbitCamera(W, H, r=1, fovy=20, convention=convention, save_path=str(tmp_path / "no_camera.json"))
    v.timestep, v.num_timesteps = timestep, T
    v.gaussians = SimpleNamespace(select_mesh_by_timestep=lambda t: None)
    v.render_buffer = np.zeros((H, W, 3), dtype=np.float32)
    v.need_update = False
    v.update_record_timeline()
    return v


def _keyframes(n, seed, intervals=None):
    """n keyframes as the viewer's get_state_dict makes them, with unequal intervals."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    rots = Rotation.random(n, random_state=seed).as_matrix()
    out = []
    for i in range(n):
        look_at = rng.normal(0.0, 0.05, 3).astype(np.float32)
        iv = int(rng.integers(3, 13)) if intervals is None else intervals[i]
        out.append(TR.keyframe(rots[i], look_at, float(rng.uniform(0.6, 1.6)), float(rng.uniform(12.0, 40.0)), iv))
    return out


def _prepare_camera(v):
    """The viewer's prepare_camera, with .cuda() a no-op (its tensors stay on the CPU)."""
    real = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        return v.prepare_camera()
    finally:
        torch.Tensor.cuda = real


CASES = [  # (keyframes, cycles, convention, W, H)
    (1, 1, "opencv", 960, 540),
    (1, 3, "opengl", 961, 541),
    (2, 0, "opencv", 960, 540),
    (2, 1, "opengl", 963, 539),
    (3, 0, "opengl", 960, 540),
    (3, 3, "opencv", 961, 541),
    (4, 0, "opencv", 965, 541),
    (4, 1, "opencv", 960, 540),
    (7, 0, "opengl", 960, 540),
    (7, 3, "opencv", 961, 543),
]


@needs_ref
@pytest.mark.parametrize("n,cycles,convention,W,H", CASES)
def test_path_equals_viewer(n, cycles, convention, W, H, tmp_path):
    kfs = _keyframes(n, seed=10 * n + cycles)
    v = _viewer(kfs, W, H, cycles, convention, tmp_path)
    path = TR.CameraPath(kfs, width=W, height=H, cycles=cycles, convention=convention)
    assert len(path) == v.num_record_timeline > 0
    assert sorted(path.states) == sorted(v.all_frames)
    for k, ref in v.all_frames.items():   # the float states, bit for bit and of the same dtype
        assert path.states[k].dtype == ref.dtype and np.array_equal(path.states[k], ref), k
    rows = path.rows()
    dpg = sys.modules["dearpygui.dearpygui"]
    for i in range(len(path)):
        dpg.set_value("_slider_record_timestep", i)
        v.apply_state_dict(v.get_state_dict_record())
        cam = _prepare_camera(v)
        assert np.array_equal(path.pose(i), v.cam.pose)
        mine = path.camera(i)
        assert (mine.FoVx, mine.FoVy) == (cam.FoVx, cam.FoVy)
        assert (mine.image_width, mine.image_height) == (cam.image_width, cam.image_height)
        assert torch.equal(rows[i], camera_block(cam, fov=True)), i


def test_keyframe_matches_get_state_dict(tmp_path):
    if not ref_import.available():
        pytest.skip("the reference is not mounted")
    from scipy.spatial.transform import Rotation
    v = _viewer([], 960, 540, 0, "opencv", tmp_path)
    v.cam.rot = Rotation.random(random_state=3)
    v.cam.look_at = np.array([0.01, -0.02, 0.03], dtype=np.float32)
    v.cam.radius, v.cam.fovy = 1.37, 23.5
    ref = v.get_state_dict()
    mine = TR.keyframe(v.cam.rot.as_matrix(), v.cam.look_at, v.cam.radius, v.cam.fovy, 25)
    for k in ref:   # the quaternion goes through the matrix: equal to rounding, up to its sign
        a, b = np.asarray(mine[k]), np.asarray(ref[k])
        assert a.dtype == b.dtype, k
        assert np.allclose(a, b, rtol=0, atol=1e-12) or (k == "rot" and np.allclose(a, -b, rtol=0, atol=1e-12)), k


@needs_ref
def test_single_keyframe_without_cycles_is_empty(tmp_path):
    kfs = _keyframes(1, seed=1)
    assert _viewer(kfs, 960, 540, 0, "opencv", tmp_path).num_record_timeline == 0
    with pytest.raises(ValueError, match="empty"):
        TR.CameraPath(kfs)


def _ref_json(T, path):
    frames = [{"timestep_index": t, "file_path": f"images/{t:05d}_{c:02d}.png",
               "fg_mask_path": f"fg_masks/{t:05d}_{c:02d}.png", "flame_param_path": f"flame_param/{t:05d}.npz"}
              for t in range(T) for c in range(2)]
    with open(path, "w") as f:
        json.dump({"frames": frames}, f)
    return path


@needs_ref
@pytest.mark.parametrize("dynamic,start,convention", [(True, 3, "opencv"), (False, 2, "opencv"), (True, 0, "opengl")])
def test_trajectory_json_equals_viewer(dynamic, start, convention, tmp_path, monkeypatch):
    """The viewer's export loop runs with its render loop replaced by a flag reset and its image save stubbed: the
    trajectory.json it writes equals CameraPath.trajectory_json, timesteps clamped at T - 1 included."""
    lv, _ = _reference()
    T = 12
    kfs = _keyframes(4, seed=5, intervals=[4, 7, 3, 5])
    ref = _ref_json(T, tmp_path / "transforms_test.json")
    v = _viewer(kfs, 961, 541, 0, convention, tmp_path, T=T, timestep=start, dynamic=dynamic, ref_json=ref)
    monkeypatch.setattr(lv, "time", SimpleNamespace(sleep=lambda s: setattr(v, "need_update", False),
                                                    strftime=lambda fmt: "export"))
    monkeypatch.setattr(lv, "Image", SimpleNamespace(fromarray=lambda a: SimpleNamespace(save=lambda p: None)))
    v.export_trajectory()
    with open(tmp_path / "viewer" / "export" / "trajectory.json") as f:
        theirs = json.load(f)
    path = TR.CameraPath(kfs, width=961, height=541, convention=convention, dynamic=dynamic, start_timestep=start,
                         num_timesteps=T)
    mine = json.loads(json.dumps(path.trajectory_json(ref)))
    assert mine == theirs
    ts = [fr["timestep_index"] for fr in mine["frames"]]
    assert ts == path.timesteps()
    if dynamic and start == 3:
        assert ts[-1] == T - 1 and ts.count(T - 1) > 1   # clamped at T - 1
    if not dynamic:
        assert set(ts) == {start}
    # without a reference json the frames carry no file-path placeholders
    plain = path.trajectory_json()
    assert all("file_path" not in fr for fr in plain["frames"])
    assert [fr["transform_matrix"] for fr in plain["frames"]] == [fr["transform_matrix"] for fr in theirs["frames"]]


def test_timesteps_static_and_dynamic():
    kfs = _keyframes(2, seed=2, intervals=[9, 1])
    assert TR.CameraPath(kfs).timesteps() is None
    p = TR.CameraPath(kfs, dynamic=True, start_timestep=5, num_timesteps=8)
    assert p.timesteps() == [5, 6, 7, 7, 7, 7, 7, 7, 7]
    assert TR.CameraPath(kfs, start_timestep=4, num_timesteps=8).timesteps() == [4] * 9


@pytest.mark.parametrize("bad,match", [
    ("empty", "at least one keyframe"),
    ("interval0", "interval must be a positive int"),
    ("interval_neg", "interval must be a positive int"),
    ("convention", "convention"),
    ("zero_quat", "zero quaternion"),
    ("missing_key", "must be a dict"),
    ("dynamic_static", "needs num_timesteps"),
    ("start", "start_timestep"),
])
def test_refusals(bad, match):
    kfs = _keyframes(3, seed=4)
    kw = {}
    if bad == "empty":
        kfs = []
    elif bad == "interval0":
        kfs[1]["interval"] = 0
    elif bad == "interval_neg":
        kfs[0]["interval"] = -3
    elif bad == "convention":
        kw["convention"] = "blender"
    elif bad == "zero_quat":
        kfs[2]["rot"] = np.zeros(4)
    elif bad == "missing_key":
        del kfs[1]["fovy"]
    elif bad == "dynamic_static":
        kw["dynamic"] = True
    elif bad == "start":
        kw.update(num_timesteps=4, start_timestep=4)
    with pytest.raises(ValueError, match=match):
        TR.CameraPath(kfs, **kw)
