"""A device-resident view schedule: which cameras, timestep and frames every iteration of a run trains or scores.

    order = epoch_order(len(records), iterations, torch.Generator().manual_seed(0))
    s = ViewSchedule(records, timesteps=ts, frames=ids, order=order)          # immutable device tensors
    frame = GraphedFrame(pc, W, H, fovx, fovy, bg, optimizer=opt, densify_stats=True, frames=store, schedule=s)
    frame.run_iterations(n)                  # n back-to-back replays, one synchronisation, no host input
    ev = GraphedEval(pc, W, H, bg, views=R * K, schedule=test, frames=store)
    ev.run_all(); ev.scores()

A record is K camera rows (`camera_block(cam, fov=True)`, 37 floats), the FLAME timestep of the model pose and the K
ids of the ground-truth frames in a FrameStore.  The order lists the record every iteration visits.  A captured frame
built with `schedule=` owns a device cursor: a sampler kernel at the head of each replay copies record order[cursor]
into the frame's static inputs, and a commit kernel at its end advances the cursor (csrc/schedule.cu).  The reference's
loop consumes its dataset exactly this way -- a DataLoader over the train cameras with shuffle=True, a fresh
permutation every epoch (train.py:55,113-116), and the test cameras in order in training_report -- so all of it is
known before the run starts and lives on the device.

Every check happens once, here or when a frame is built on the schedule: the order's entries index the records, the
timesteps the model's, the ids the store's frames, and the cameras have the frame's image size.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _native as N

CAMERA_FLOATS = N.CAMERA_FLOATS


def epoch_order(records: int, iterations: int, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """(iterations,) int32: one torch.randperm(records, generator=generator) per epoch, concatenated and truncated to
    `iterations` -- the per-epoch permutations of the reference's DataLoader(shuffle=True).  It does not reproduce the
    DataLoader's own random stream (which draws its permutations from its own generator): the same seed gives another
    order than the reference's, with the same semantics (every record once per epoch, a fresh order per epoch)."""
    records, iterations = int(records), int(iterations)
    if records < 1 or iterations < 0:
        raise ValueError(f"epoch_order needs records >= 1 and iterations >= 0, got {records}, {iterations}")
    parts, n = [], 0
    while n < iterations:
        parts.append(torch.randperm(records, generator=generator))
        n += records
    if not parts:
        return torch.zeros(0, dtype=torch.int32)
    return torch.cat(parts)[:iterations].to(torch.int32)


def _cuda_device(device) -> torch.device:
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("gaussianavatars_b200 has no CPU path: a ViewSchedule lives on a CUDA device")
    return dev


def _int_table(values, shape, name) -> torch.Tensor:
    t = torch.as_tensor(values)
    if t.dtype.is_floating_point or t.dtype == torch.bool or t.dtype.is_complex:
        raise ValueError(f"{name} must hold integers, got {t.dtype}")
    if t.numel() != int(torch.tensor(shape).prod()):
        raise ValueError(f"{name} must hold {'x'.join(map(str, shape))} values, got {tuple(t.shape)}")
    t = t.reshape(shape).to(torch.int64)
    if t.numel() and (int(t.min()) < 0 or int(t.max()) > 2 ** 31 - 1):
        raise ValueError(f"{name} must be non-negative int32 values")
    return t.to(torch.int32)


class ViewSchedule:
    def __init__(self, cameras, timesteps=None, frames=None, order=None, device=None):
        """cameras: R camera objects (K = 1), R groups of K camera objects, or a float tensor (R, K, 37) / (R, 37) of
        camera_block(cam, fov=True) rows.  Every camera object must have one image size (`W`, `H`; None for a
        tensor, whose size the caller vouches for).
        timesteps: R ints (the FLAME timestep of every record), required by a model with a FLAME head and refused by
        one without.  frames: R ids (K = 1) or (R, K) ids of a FrameStore, required by a frame that reads one.
        order: L record indices in [0, R), the record of iteration i (default: the identity, which evaluation wants;
        epoch_order gives the training loader's).  device: a CUDA device (default: the tensor's, else the current)."""
        from .graph import camera_block
        from .renderer import camera_table
        self.W = self.H = None
        if isinstance(cameras, torch.Tensor):
            cams = cameras.detach()
            if cams.dim() == 2:
                cams = cams.unsqueeze(1)
            if cams.dim() != 3 or cams.shape[0] < 1 or cams.shape[1] < 1 or cams.shape[2] != CAMERA_FLOATS:
                raise ValueError(f"a camera tensor of a schedule is (R, K, {CAMERA_FLOATS}) or (R, {CAMERA_FLOATS}), "
                                 f"got {tuple(cameras.shape)}")
            if device is None and cams.device.type == "cuda":
                device = cams.device
        else:
            recs = list(cameras)
            if not recs:
                raise ValueError("a schedule holds at least one record")
            grouped = not hasattr(recs[0], "world_view_transform")
            groups = [list(g) for g in recs] if grouped else [[c] for c in recs]
            K = len(groups[0])
            if K < 1 or any(len(g) != K for g in groups):
                raise ValueError(f"every record of a schedule has the same number of cameras, got "
                                 f"{sorted({len(g) for g in groups})}")
            sizes = {(int(c.image_width), int(c.image_height)) for g in groups for c in g}
            if len(sizes) != 1:
                raise ValueError(f"the cameras of a schedule have one image size, got {sorted(sizes)}")
            (self.W, self.H), = sizes
            # the rows a host-driven frame would write: camera_block for one view, camera_table for K views
            cams = torch.stack([camera_block(g[0], fov=True).unsqueeze(0) if not grouped else camera_table(g, "cpu")
                                for g in groups])
        if not 1 <= cams.shape[1] <= N.MAX_VIEWS:
            raise ValueError(f"a record holds 1 .. {N.MAX_VIEWS} cameras, got {cams.shape[1]}")
        self.device = _cuda_device(device)
        self.R, self.K = int(cams.shape[0]), int(cams.shape[1])
        if self.R * self.K > 2 ** 31 - 1:
            raise ValueError("a schedule holds at most 2^31 - 1 camera rows")
        if not torch.isfinite(cams).all():
            raise ValueError("the camera rows of a schedule must be finite")
        self.cams = cams.to(self.device, torch.float32).contiguous()
        self.timesteps = self.frame_ids = self.timesteps_host = None
        self.max_timestep = self.max_frame_id = None
        if timesteps is not None:
            t = _int_table(timesteps, (self.R,), "timesteps")
            self.max_timestep = int(t.max())
            self.timesteps_host = t.tolist()
            self.timesteps = t.to(self.device).contiguous()
        if frames is not None:
            f = _int_table(frames, (self.R, self.K), "frames")
            self.max_frame_id = int(f.max())
            self.frame_ids = f.to(self.device).contiguous()
        o = torch.arange(self.R) if order is None else torch.as_tensor(order)
        if o.dtype.is_floating_point or o.dtype == torch.bool or o.dim() != 1 or o.numel() < 1:
            raise ValueError("order must be a non-empty 1-D sequence of record indices")
        if int(o.min()) < 0 or int(o.max()) >= self.R:
            raise ValueError(f"order entries index the schedule's {self.R} records: got values in "
                             f"[{int(o.min())}, {int(o.max())}]")
        self.L = int(o.numel())
        self.order = o.to(torch.int32).to(self.device).contiguous()
        self.order_host = o.to(torch.int64).tolist()
        for t in (self.cams, self.timesteps, self.frame_ids, self.order):   # immutable: a replay reads them by address
            if t is not None:
                t.requires_grad_(False)

    def __len__(self) -> int:
        return self.L

    def record(self, i: int) -> int:
        """The record iteration i visits (a host lookup)."""
        return self.order_host[i]

    def warm_records(self, n: int = 16) -> list:
        """Up to n record indices spread evenly over the table: the records a frame built on the schedule renders
        eagerly to size its instance capacity (each at its own timestep)."""
        n = min(int(n), self.R)
        return sorted({round(i * (self.R - 1) / max(n - 1, 1)) for i in range(n)})

    def check_for(self, consumer: str, W: int, H: int, K: int, device, num_timesteps: Optional[int], store) -> None:
        """The checks of a frame built on this schedule: its image size, views per replay and device; timesteps exactly
        when the model has a FLAME head (within its num_timesteps); ids exactly when it reads a store (within
        len(store))."""
        if self.K != K:
            raise ValueError(f"the schedule's records hold {self.K} cameras, this {consumer} renders {K} per replay")
        if self.W is not None and (self.W, self.H) != (W, H):
            raise ValueError(f"the schedule's cameras are {self.W}x{self.H}, this {consumer} renders {W}x{H}")
        if self.device != torch.device(device):
            raise ValueError(f"the schedule lives on {self.device}, this {consumer} on {device}")
        if num_timesteps is None and self.timesteps is not None:
            raise ValueError("the schedule carries timesteps, but the model has no FLAME head to pose with them")
        if num_timesteps is not None:
            if self.timesteps is None:
                raise ValueError("the model poses a FLAME head: the schedule needs timesteps=")
            if self.max_timestep >= num_timesteps:
                raise ValueError(f"the schedule's timesteps reach {self.max_timestep}, the model has {num_timesteps}")
        if store is None and self.frame_ids is not None:
            raise ValueError(f"the schedule carries frame ids, but this {consumer} reads no frame store (frames=)")
        if store is not None:
            if self.frame_ids is None:
                raise ValueError("a frame that reads a frame store needs a schedule with frames=")
            if self.max_frame_id >= len(store):
                raise ValueError(f"the schedule's frame ids reach {self.max_frame_id}, the store holds {len(store)} "
                                 "frames")
