"""The reference local viewer's recorded camera paths (local_viewer.py's Record panel), played on the device.

    path = CameraPath([keyframe(R0, look_at0, 1.0, 20.0), keyframe(R1, look_at1, 1.2, 20.0)],
                      width=960, height=540, dynamic=True, num_timesteps=T)
    export_trajectory(pc, path, "out/", bg=bg, mesh_opacity=0.5, video="out/path.mp4")

A keyframe is the viewer's state dict: `rot` (an xyzw quaternion), `look_at`, `radius`, `fovy` (degrees) and
`interval` (frames to the next keyframe).  CameraPath restates the viewer's timeline (update_record_timeline): the
frames between keyframes are interpolated per component with scipy's interp1d -- linear for two or three keyframes,
cubic for four or more, `fill_value='extrapolate'` -- and every frame's state is applied to an orbit camera exactly as
the viewer applies it (apply_state_dict, OrbitCamera.pose / world_view_transform / projection_from_intrinsics / fovx,
prepare_camera).  The float64 states and the float32 camera rows are the viewer's own, bit for bit, because the same
numpy and scipy operations compute them.

`schedule(device)` turns the path into a schedule.ViewSchedule with the identity order: a GraphedRender built with
`schedule=` plays it as back-to-back replays, each taking its camera row and timestep from the device cursor.
`export_trajectory` writes what the viewer's "export traj" button writes -- the PNG frames 00000.png ... and
trajectory.json -- and optionally an MP4, with the frames quantised as the viewer quantises them
(GraphedRender(quantize="viewer")).

Only this module imports scipy.
"""
from __future__ import annotations

import json
import math
import os
from types import SimpleNamespace
from typing import Optional, Sequence

import numpy as np
import torch

CONVENTIONS = ("opencv", "opengl")
_STATE_KEYS = ("rot", "look_at", "radius", "fovy", "interval")


def keyframe(rotation, look_at, radius: float, fovy: float, interval: int = 25) -> dict:
    """A keyframe as the viewer's get_state_dict makes it from an OrbitCamera: rotation a 3x3 rotation matrix (the
    camera's OpenGL-convention orientation, OrbitCamera.rot.as_matrix()), look_at (3,), radius, fovy in degrees and
    the interval to the next keyframe in frames (the viewer's fps * keyframe_interval)."""
    from scipy.spatial.transform import Rotation
    return {
        "rot": Rotation.from_matrix(np.asarray(rotation)).as_quat(),
        "look_at": np.array(look_at),
        "radius": np.array([radius]).astype(np.float32),
        "fovy": np.array([fovy]).astype(np.float32),
        "interval": int(interval),
    }


def _check_keyframe(i: int, kf) -> dict:
    if not isinstance(kf, dict) or any(k not in kf for k in _STATE_KEYS):
        raise ValueError(f"keyframe {i} must be a dict with {', '.join(_STATE_KEYS)} (trajectory.keyframe builds one)")
    interval = kf["interval"]
    if isinstance(interval, bool) or not isinstance(interval, (int, np.integer)) or interval < 1:
        raise ValueError(f"keyframe {i}: interval must be a positive int, got {interval!r}")
    rot = np.asarray(kf["rot"], dtype=np.float64)
    if rot.shape != (4,) or not np.isfinite(rot).all():
        raise ValueError(f"keyframe {i}: rot must be 4 finite values (an xyzw quaternion), got {rot.shape}")
    if not np.linalg.norm(rot) > 0.0:
        raise ValueError(f"keyframe {i}: rot is the zero quaternion, which is no rotation")
    for k, n in (("look_at", 3), ("radius", 1), ("fovy", 1)):
        v = np.asarray(kf[k], dtype=np.float64)
        if v.size != n or not np.isfinite(v).all():
            raise ValueError(f"keyframe {i}: {k} must be {n} finite value(s), got {v.shape}")
    return kf


class CameraPath:
    def __init__(self, keyframes: Sequence[dict], width: int = 960, height: int = 540, cycles: int = 0,
                 convention: str = "opencv", znear: float = 0.01, zfar: float = 10.0, dynamic: bool = False,
                 start_timestep: int = 0, num_timesteps: Optional[int] = None):
        """keyframes: the viewer's keyframe state dicts, in order (keyframe() builds one).  width / height: the
        viewer's window (960x540 by default).  cycles: the viewer's "cycles" field (0: from the first keyframe to the
        last; n > 0: n loops through all keyframes, the list padded with one extra loop at each end).  convention:
        the viewer's cam_convention, "opencv" (its default) or "opengl"; znear / zfar: the OrbitCamera's.
        num_timesteps: T of a model with a FLAME head (None: a static model; the schedule then carries no
        timesteps).  dynamic: the viewer's "dynamic" checkbox -- frame i is rendered at min(start_timestep + i, T - 1);
        without it every frame is at start_timestep."""
        kfs = [_check_keyframe(i, kf) for i, kf in enumerate(keyframes)]
        if not kfs:
            raise ValueError("a camera path needs at least one keyframe")
        if convention not in CONVENTIONS:
            raise ValueError(f"convention must be 'opencv' or 'opengl', got {convention!r}")
        if isinstance(cycles, bool) or not isinstance(cycles, int) or cycles < 0:
            raise ValueError(f"cycles must be an int >= 0, got {cycles!r}")
        W, H = int(width), int(height)
        if W < 1 or H < 1:
            raise ValueError(f"the image size must be positive, got {W}x{H}")
        if num_timesteps is not None:
            num_timesteps = int(num_timesteps)
            if num_timesteps < 1 or not 0 <= int(start_timestep) < num_timesteps:
                raise ValueError(f"start_timestep must lie in [0, {num_timesteps}), got {start_timestep}")
        elif dynamic:
            raise ValueError("dynamic=True advances the FLAME timestep: it needs num_timesteps")
        self.keyframes, self.W, self.H, self.cycles = kfs, W, H, cycles
        self.convention, self.znear, self.zfar = convention, float(znear), float(zfar)
        self.dynamic, self.start_timestep, self.num_timesteps = bool(dynamic), int(start_timestep), num_timesteps
        self.num_frames, self.states = self._timeline()
        if self.num_frames < 1:
            raise ValueError("the camera path is empty: with cycles=0 it runs from the first keyframe to the last, so it "
                             "needs two keyframes (or cycles > 0)")

    # ---- the viewer's timeline (update_record_timeline) ---------------------------------------------------------
    def _timeline(self):
        from scipy.interpolate import interp1d
        own, cycles = self.keyframes, self.cycles
        if cycles == 0:
            n = sum([kf["interval"] for kf in own[:-1]])
        else:
            n = sum([kf["interval"] for kf in own]) * cycles
        kfs = list(own)
        if cycles > 0:   # one extra loop at each end, so that the spline runs smoothly through the first and last
            kfs = own * (cycles + 2)
            t = -sum([kf["interval"] for kf in own])
        else:
            t = 0
        k_x = []
        for kf in kfs:
            k_x.append(t)
            t += kf["interval"]
        x = np.arange(n)
        states = {}
        if len(kfs) <= 1:
            for k in kfs[0]:
                k_y = np.concatenate([np.array(kf[k])[None] for kf in kfs], axis=0)
                states[k] = np.tile(k_y, (n, 1))
        else:
            kind = "linear" if len(kfs) <= 3 else "cubic"
            for k in kfs[0]:
                if k == "interval":
                    continue
                k_y = np.concatenate([np.array(kf[k])[None] for kf in kfs], axis=0)
                funcs = [interp1d(k_x, k_y[:, i], kind=kind, fill_value="extrapolate") for i in range(k_y.shape[1])]
                states[k] = np.array([f(x) for f in funcs]).transpose(1, 0)
        return int(n), states

    def __len__(self) -> int:
        return self.num_frames

    def state(self, i: int) -> dict:
        """Frame i's interpolated state dict (the viewer's get_state_dict_record)."""
        return {k: self.states[k][i] for k in self.states}

    def timestep(self, i: int) -> Optional[int]:
        """The FLAME timestep of frame i (None for a static model)."""
        if self.num_timesteps is None:
            return None
        if not self.dynamic:
            return self.start_timestep
        return min(self.start_timestep + i, self.num_timesteps - 1)

    def timesteps(self) -> Optional[list]:
        return None if self.num_timesteps is None else [self.timestep(i) for i in range(self.num_frames)]

    # ---- the viewer's orbit camera (apply_state_dict, OrbitCamera, prepare_camera) ------------------------------
    def _orbit(self, i: int) -> SimpleNamespace:
        """Frame i's camera state after apply_state_dict: rot (a scipy Rotation), look_at, radius, fovy."""
        from scipy.spatial.transform import Rotation
        st = self.state(i)
        try:
            rot = Rotation.from_quat(st["rot"])
        except ValueError as e:   # an interpolated quaternion can pass through zero
            raise ValueError(f"frame {i}: the interpolated rotation is not a rotation ({e})") from None
        return SimpleNamespace(rot=rot, look_at=st["look_at"], radius=st["radius"].item(), fovy=st["fovy"].item())

    def _intrinsics(self, fovy):
        focal = self.H / (2 * np.tan(np.radians(fovy) / 2))
        return np.array([focal, focal, self.W // 2, self.H // 2])

    def pose(self, i: int) -> np.ndarray:
        """(4,4) float32 camera-to-world of frame i in the path's convention (OrbitCamera.pose)."""
        o = self._orbit(i)
        pose = np.eye(4, dtype=np.float32)
        pose[2, 3] += o.radius
        rot = np.eye(4, dtype=np.float32)
        rot[:3, :3] = o.rot.as_matrix()
        pose = rot @ pose
        pose[:3, 3] -= o.look_at
        if self.convention == "opencv":
            pose[:, [1, 2]] *= -1
        return pose

    def _projection(self, fovy) -> np.ndarray:
        K = self._intrinsics(fovy)[None]
        z_sign = 1 if self.convention == "opencv" else -1
        near, far = self.znear, self.zfar
        proj = np.zeros([1, 4, 4])
        proj[:, 0, 0] = K[..., [0]] * 2 / self.W
        proj[:, 1, 1] = K[..., [1]] * 2 / self.H
        proj[:, 0, 2] = (self.W - 2 * K[..., [2]]) / self.W
        proj[:, 1, 2] = (self.H - 2 * K[..., [3]]) / self.H
        proj[:, 2, 2] = z_sign * (far + near) / (far - near)
        proj[:, 2, 3] = -2 * far * near / (far - near)
        proj[:, 3, 2] = z_sign
        return proj[0]

    def _fovx(self, fovy) -> float:
        focal = self.H / (2 * np.tan(np.radians(fovy) / 2))
        return np.degrees(2 * np.arctan(self.W / (2 * focal)))

    def camera(self, i: int) -> SimpleNamespace:
        """Frame i's camera as the viewer hands it to render() (prepare_camera), with CPU tensors."""
        fovy = self._orbit(i).fovy
        pose = self.pose(i)
        wvt = np.linalg.inv(pose)
        full = self._projection(fovy) @ wvt
        return SimpleNamespace(
            FoVx=float(np.radians(self._fovx(fovy))), FoVy=float(np.radians(fovy)),
            image_height=self.H, image_width=self.W,
            world_view_transform=torch.tensor(wvt).float().T, full_proj_transform=torch.tensor(full).float().T,
            camera_center=torch.tensor(pose[:3, 3]))

    def rows(self) -> torch.Tensor:
        """(L, 37) float32: every frame's camera_block(camera(i), fov=True), the rows a GraphedRender renders."""
        from .graph import camera_block
        return torch.stack([camera_block(self.camera(i), fov=True) for i in range(self.num_frames)])

    def schedule(self, device=None):
        """A schedule.ViewSchedule of the path's frames in order (the identity order), with their timesteps when the
        path has num_timesteps."""
        from .schedule import ViewSchedule
        return ViewSchedule([self.camera(i) for i in range(self.num_frames)], timesteps=self.timesteps(),
                            device=device)

    # ---- trajectory.json (export_trajectory) ---------------------------------------------------------------------
    def trajectory_json(self, ref_json=None) -> dict:
        """The dict the viewer's export writes as trajectory.json: per frame the intrinsics, the OpenGL
        camera-to-world `transform_matrix`, `timestep_index` and `camera_indx`, then the sorted `timestep_indices`
        and `camera_indices`.  ref_json (a path, or the loaded dict, of a dataset's transforms json): each frame also
        gets the file_path, fg_mask_path and flame_param_path of the reference's first frame at its timestep, as
        placeholders that let render.py load the trajectory like a sequence (a timestep the reference lacks gets
        none)."""
        tid2paths = {}
        if ref_json is not None:
            if not isinstance(ref_json, dict):
                with open(ref_json, "r") as f:
                    ref_json = json.load(f)
            for frame in ref_json["frames"]:
                tid = frame["timestep_index"]
                if tid not in tid2paths:
                    tid2paths[tid] = frame
        traj = {"frames": []}
        timestep_indices, camera_indices = [], []
        for i in range(self.num_frames):
            intr = self._intrinsics(self._orbit(i).fovy)
            cx, cy = intr[2], intr[3]
            fl_x, fl_y = intr[0], intr[1]
            h, w = self.H, self.W
            c2w = self.pose(i).copy()   # the viewer's export assumes the opencv convention here
            c2w[:, [1, 2]] *= -1
            t = self.timestep(i)
            timestep_index = 0 if t is None else t
            timestep_indices.append(timestep_index)
            camera_indices.append(i)
            frame = {"cx": cx, "cy": cy, "fl_x": fl_x, "fl_y": fl_y, "h": h, "w": w,
                     "camera_angle_x": math.atan(w / (fl_x * 2)) * 2, "camera_angle_y": math.atan(h / (fl_y * 2)) * 2,
                     "transform_matrix": c2w.tolist(), "timestep_index": timestep_index, "camera_indx": i}
            if timestep_index in tid2paths:
                for k in ("file_path", "fg_mask_path", "flame_param_path"):
                    frame[k] = tid2paths[timestep_index][k]
            traj["frames"].append(frame)
        traj["timestep_indices"] = sorted(list(set(timestep_indices)))
        traj["camera_indices"] = sorted(list(set(camera_indices)))
        return traj


@torch.no_grad()
def export_trajectory(pc, path: CameraPath, out_dir, *, bg: torch.Tensor, mesh_opacity: Optional[float] = None,
                      face_colors: Optional[torch.Tensor] = None, scaling_modifier: float = 1.0, video=None,
                      gop: int = 25, fps: int = 25, qp: int = 20, batch: int = 16, ref_json=None,
                      capacity: Optional[int] = None, deblock: bool = False, intra4x4: bool = False) -> dict:
    """What the viewer's "export traj" button writes, rendered on the device: out_dir/00000.png ... (one PNG per frame
    of the path, the viewer's bytes: GraphedRender(quantize="viewer", png=True)) and out_dir/trajectory.json
    (path.trajectory_json(ref_json)).  mesh_opacity: the viewer's "show mesh" at that opacity (its default colour
    alpha is 0.5), face_colors its face colours; scaling_modifier its "Scale modifier" slider.  video: a file name or
    binary file object, also written as an MP4 of the same frames (video.VideoWriter at fps, qp, gop, deblock and
    intra4x4).

    The frames are played by one scheduled GraphedRender, `batch` replays at a time with no host input; each batch
    ends in one synchronisation, after which its PNG files are written from the pinned ring and its frames join the
    video.  A batch in which a replay overflowed the instance capacity is played again after the graph regrew.
    capacity: the initial instance capacity (default: sized by eager frames over the path).  Returns
    {"frames": L, "captures": re-captures, "trajectory": the json dict}."""
    from .graph import GraphedRender
    from .video import VideoWriter
    if isinstance(batch, bool) or not isinstance(batch, int) or batch < 1:
        raise ValueError(f"batch must be a positive int, got {batch!r}")
    if not isinstance(deblock, bool):
        raise ValueError(f"deblock must be a bool, got {deblock!r}")
    if not isinstance(intra4x4, bool):
        raise ValueError(f"intra4x4 must be a bool, got {intra4x4!r}")
    num_timesteps = int(pc.flame_param["expr"].shape[0]) if getattr(pc, "flame", None) is not None else None
    if (path.num_timesteps is None) != (num_timesteps is None):
        raise ValueError("the path carries FLAME timesteps exactly when the model has a FLAME head: build it with "
                         f"num_timesteps={num_timesteps}")
    if num_timesteps is not None and path.num_timesteps != num_timesteps:
        raise ValueError(f"the path was built for {path.num_timesteps} timesteps, the model has {num_timesteps}")
    traj = path.trajectory_json(ref_json)
    os.makedirs(out_dir, exist_ok=True)
    device = pc._xyz.device
    sched = path.schedule(device)
    L = len(sched)
    B = min(batch, L)
    view = GraphedRender(pc, path.W, path.H, bg, outputs="u8", scaling_modifier=scaling_modifier, host_slots=B,
                         capacity=capacity, mesh_opacity=mesh_opacity, face_colors=face_colors, png=True,
                         quantize="viewer", schedule=sched)
    writer = VideoWriter(video, path.W, path.H, fps=fps, qp=qp, batch=B, device=device, gop=gop, deblock=deblock,
                         intra4x4=intra4x4) if video is not None else None
    frames = torch.empty((B, path.H, path.W, 3), dtype=torch.uint8, device=device) if writer is not None else None
    try:
        view.capture()
        done = 0
        while done < L:
            n = min(B, L - done)
            view.set_cursor(done)
            first = view.replays
            for j in range(n):
                view.run_iterations(1, check=False)
                if frames is not None:
                    frames[j].copy_(view.display)
            if view.overflowed(wait=True):   # the batch's one synchronisation
                view.regrow(int(view.cursor.item()))   # the record that overflowed joins the warm-up
                continue   # play the batch again at the grown capacity
            for j in range(n):
                with open(os.path.join(out_dir, f"{done + j:05d}.png"), "wb") as f:
                    f.write(view.host_png(first + j))
            if writer is not None:
                writer.add(frames[:n])
            done += n
    finally:
        if writer is not None:
            writer.close()
    with open(os.path.join(out_dir, "trajectory.json"), "w") as f:
        json.dump(traj, f, indent=4)
    return {"frames": L, "captures": view.captures, "trajectory": traj}
