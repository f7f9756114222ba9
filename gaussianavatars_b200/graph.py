"""One training frame of the hot path as ONE CUDA graph.

    frame = GraphedFrame(pc, width, height, fovx, fovy, bg, loss="l1_u8")
    frame.set_inputs(camera=cam, verts=posed_vertices, gt_u8=ground_truth)     # device or pinned-host tensors
    frame.run()                                                                # enqueue one replay
    pc._xyz.grad, frame.verts.grad, frame.loss ...                             # static result tensors

By default the field of view is the `fovx`/`fovy` given at construction, baked into the graph: every replay renders
with it, so that mode is only correct for cameras that share one FoV.  With `per_camera_fov=True` the camera block
also carries tan(FoVx/2), tan(FoVy/2) (`camera_block(cam, fov=True)`, 37 floats) and the kernels read them from device
memory on every replay: one captured graph trains every camera of a calibrated rig (the reference gives each camera
its own FoV, scene/dataset_readers.py).

What is captured (the data flow of the reference training step, train.py:113-170, with the fused route of
`render()`): [H2D copy of the camera block and the uint8 ground truth] -> per-face frame of the posed mesh
(scene/flame_gaussian_model.py:137-147) -> fused binding + rasterizer forward (gaussian_renderer/__init__.py:19-101) ->
loss (utils/loss_utils.py:17-63) -> backward down to the raw splat parameters and the mesh vertices -> [D2H copy of
the loss scalar].  ~25 launches, memsets and copies become one `cudaGraphLaunch`: the host is off the step.

The forward inside the graph runs with `GAB200_SYNC_NONE` (include/gab200_rasterizer.h): the instance capacity is
fixed at capture time from the frames rendered eagerly before it (x `headroom`).  A replay that needs more than the
capacity renders from a truncated instance list -- memory-safe, wrong -- and raises the slot's sticky device flag;
`run(check=True)` waits for the replay, and on overflow grows the capacity, re-captures and replays: its results are
then exactly those of an eager `render()`.  `run(check=False)` never touches the host; call `overflowed()` whenever
convenient (bench.py does after its timed loop).

With `optimizer=` (a capturable `Adam`) and `densify_stats=True` one replay is a whole training iteration of the
reference (train.py:106-210): after backward the graph also accumulates the densification statistics
(densify.add_densification_stats) and steps the optimizer, learning-rate schedule included (training.expon_lr_schedule).
Both are skipped on the device when the replay overflowed its capacity: such a replay changes no parameter, moment,
step or statistic.  densify_and_prune / reset_opacity / oneupSHdegree stay eager calls between replays; `run()` notices
the tensors or sizes they replaced and re-captures.

When the model carries a FLAME head (`pc.flame`, a flame.FlameLBS, and `pc.flame_param`), the captured frame starts
from the pose of the reference (select_mesh_by_timestep, scene/flame_gaussian_model.py:117-135) instead of given
vertices: `set_inputs(timestep=t)` writes t into a device int32 that the replay reads, so changing the timestep never
re-captures.  The gradients reach the FLAME tensors, and a capturable `Adam` holding their groups
(flame.flame_param_groups) steps them in the same replay.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import torch

from . import _native as N
from . import mesh as M
from . import rasterizer as R
from types import SimpleNamespace

from .renderer import _forward_only, camera_table, render, render_views_train
from .rasterizer import l1_loss_u8
from .densify import add_densification_stats
from .training import (METRIC_NAMES, Adam, binding_regularizers, launch_composite_rgba, launch_image_metrics,
                       metrics_scratch, photometric_loss)
from .flame import check_timestep, flame_pose
from .lpips import LpipsNet, launch_lpips, lpips_scratch
from . import png as PNG

_STATS = ("xyz_gradient_accum", "denom", "max_radii2D")
_FLAME_KEYS = ("shape", "static_offset", "expr", "rotation", "neck_pose", "jaw_pose", "eyes_pose", "translation")


class _Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


class _GraphCamera:
    """Camera whose matrices (and, in a 37-float block, device field of view `tanfov`) are views into the graph's
    static camera block."""

    def __init__(self, W, H, fovx, fovy, block):
        self.image_width, self.image_height, self.FoVx, self.FoVy = W, H, fovx, fovy
        self.world_view_transform = block[0:16].view(4, 4)
        self.full_proj_transform = block[16:32].view(4, 4)
        self.camera_center = block[32:35]
        self.tanfov = block[35:37] if block.numel() == CAMERA_BLOCK_FOV else None


CAMERA_BLOCK, CAMERA_BLOCK_FOV = 35, 37


def tanfov_floats(fovx: float, fovy: float) -> torch.Tensor:
    """(2,) float32 {tan(fovx/2), tan(fovy/2)}: computed in double and rounded once, as render()'s settings round
    them on their way to the kernels."""
    return torch.tensor([math.tan(fovx * 0.5), math.tan(fovy * 0.5)], dtype=torch.float32)


def camera_block(cam, fov: bool = False) -> torch.Tensor:
    """(35,) float32: world_view_transform (16) | full_proj_transform (16) | camera_center (3) of a camera object.
    fov=True: (37,), followed by tan(FoVx/2), tan(FoVy/2) (a GraphedFrame with per_camera_fov=True)."""
    parts = [cam.world_view_transform.reshape(-1).float(), cam.full_proj_transform.reshape(-1).float(),
             cam.camera_center.reshape(-1).float()]
    if fov:
        parts.append(tanfov_floats(cam.FoVx, cam.FoVy).to(parts[0].device))
    return torch.cat(parts)


def pair_with_deferred_reduce(frames, buffers, side_work_at: str = "start"):
    """Two frames of one model used alternately, each with its own caller-owned gradient buffer
    (dist.SymmetricGradBuffer, mode "two_shot" or "plain"): frame k's backward fills buffers[k], and a forked branch of
    frame k's graph all-reduces buffers[1-k] -- the gradients of the PREVIOUS step -- while frame k computes.  After
    replay i the reduced gradients of step i-1 are in buffers[1-k] (`reduced_grads(frames, buffers, k)`), those of
    step i become available after replay i+1 or `buffers[k].reduce()`.  The collective leaves the critical path; the
    price is that an optimizer consuming reduced gradients runs one replay behind (DESIGN.md section 6).
    Call before capture()."""
    if len(frames) != 2 or len(buffers) != 2:
        raise ValueError("a deferred-reduction pair is two frames and two buffers")
    if any(f.optimizer is not None for f in frames):
        raise ValueError("a deferred-reduction pair reduces each step's gradients one replay late: a frame of the pair "
                         "cannot step an optimizer inside its graph")
    for k, f in enumerate(frames):
        mine, other = buffers[k], buffers[1 - k]

        def before(f=f, mine=mine):
            f.pc.symm_grad = mine
            mine.begin()

        f.before_backward = before
        f.after_backward = lambda mine=mine: mine.end(reduce=False)
        f.side_work = other.reduce
        f.side_work_at = side_work_at
        if f._side is None:
            f._side = torch.cuda.Stream(device=f.device)
    return frames


def reduced_grads(buffers, k):
    """Views (in pc.parameters() order) of the all-reduced gradients available after replaying frame k of a
    deferred-reduction pair: those of the step before."""
    return buffers[1 - k].all_views[0]


def _check_views_per_replay(k):
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= N.MAX_VIEWS:
        raise ValueError(f"views_per_replay must be an int in [1, {N.MAX_VIEWS}]")


class _Captured:
    """What a frame captured into one CUDA graph owns, whether it trains (GraphedFrame) or plays back (GraphedRender):
    the static camera block, the pose input (a device FLAME timestep, or vertices), the instance capacity -- sized by
    eager warm-up frames, guarded by the sticky overflow flag of the capture slot, grown by regrow() -- and the key of
    what the capture baked in, which run() compares to know when to re-capture.  A subclass provides `_body(captured)`,
    `_release()` (drop what the warm-up frames left behind), `_before_capture()` and `_after_capture()`, and extends
    `_state_key()` with what only its own capture bakes in."""

    K = 1   # cameras per replay (views_per_replay); a subclass sets it before __init__
    schedule = None   # a schedule.ViewSchedule the replays follow (_use_schedule)

    def __init__(self, pc, width, height, fovx, fovy, bg, per_camera_fov, capacity, headroom, warm_cameras,
                 warm_timesteps=None, verts_grad=False):
        self.pc, self.W, self.H, self.fovx, self.fovy = pc, int(width), int(height), float(fovx), float(fovy)
        self.per_camera_fov = bool(per_camera_fov)
        self.headroom, self._capacity = float(headroom), capacity
        dev = pc._xyz.device
        self.device = dev
        self.bg = bg.to(dev).float().contiguous()
        self.K = getattr(self, "K", 1)   # cameras per replay (GraphedRender(views_per_replay=K)): a (K, 37) table
        nblk = CAMERA_BLOCK_FOV if self.per_camera_fov else CAMERA_BLOCK
        self.cam = torch.zeros((self.K, nblk) if self.K > 1 else nblk, dtype=torch.float32, device=dev)
        if self.per_camera_fov:
            self.cam[..., CAMERA_BLOCK:] = tanfov_floats(self.fovx, self.fovy).to(dev)
        self.camera = _GraphCamera(self.W, self.H, self.fovx, self.fovy, self.cam) if self.K == 1 else None
        self.flame = getattr(pc, "flame", None)
        if self.flame is not None:   # the pose is computed inside the graph from this timestep
            self.verts, self.timestep = None, torch.zeros(1, dtype=torch.int32, device=dev)
            self.num_timesteps = int(pc.flame_param["expr"].shape[0])
        else:   # verts_grad: the backward reaches the vertices, which the model must then have
            rest = pc.verts_rest if verts_grad else getattr(pc, "verts_rest", None)
            self.verts = None if rest is None else rest.detach().clone().contiguous().requires_grad_(verts_grad)
            self.timestep = None
        self._warm = None if warm_cameras is None else [self._camera_tensor(c) for c in warm_cameras]
        self._warm_t = None if warm_timesteps is None or self.flame is None else [int(t) for t in warm_timesteps]
        self._warm_pairs = None   # (block, timestep) pairs rendered in place of the warm cameras x warm timesteps
        self.graph = self.slot = self._key = None
        self.replays = self.captures = 0
        self._side = None                    # copy stream of host-input uploads (a subclass creates it)
        self._gt_ready = self._done = None   # events ordering an upload against the replays that read its buffer

    def _camera_tensor(self, camera):
        """A camera object or block as this frame's block: 37 floats with per_camera_fov, else as given.  A frame of K > 1
        views per replay: a group of K camera objects (one image size) or a (K, 37) table."""
        if self.K > 1:
            if isinstance(camera, torch.Tensor):
                if tuple(camera.shape) != (self.K, CAMERA_BLOCK_FOV):
                    raise ValueError(f"a camera table of this frame is ({self.K}, {CAMERA_BLOCK_FOV}), got "
                                     f"{tuple(camera.shape)}")
                return camera.float()
            cams = list(camera)
            if len(cams) != self.K:
                raise ValueError(f"this frame renders {self.K} cameras per replay, got {len(cams)}")
            return camera_table(cams, self.device)
        blk = camera if isinstance(camera, torch.Tensor) else camera_block(camera, fov=self.per_camera_fov)
        if self.per_camera_fov and blk.numel() != CAMERA_BLOCK_FOV:
            raise ValueError(f"a {type(self).__name__} camera block with the field of view has {CAMERA_BLOCK_FOV} "
                             f"floats (camera_block(cam, fov=True)), got {blk.numel()}")
        return blk

    def _gt_shape(self):
        return (3, self.H, self.W) if self.K == 1 else (self.K, 3, self.H, self.W)

    def _set_pose_input(self, verts, timestep):
        """The checks of set_inputs' pose arguments; writes the timestep (a host int checked against the model's
        number of timesteps) into the device int32 the replay reads."""
        if verts is not None and self.flame is not None:
            raise ValueError("this frame poses its FLAME head itself: give set_inputs(timestep=...), not verts")
        if timestep is not None:
            if self.flame is None:
                raise ValueError("timestep= needs a model with a FLAME head (pc.flame)")
            self.timestep.fill_(check_timestep(timestep, self.num_timesteps))

    def _pose(self):
        """The model's face frame from the FLAME pose of the device timestep, or from the given vertices."""
        pc = self.pc
        if self.flame is not None:
            verts, pc.verts_cano = flame_pose(self.flame, pc.flame_param, self.timestep)
            pc.update_mesh_properties(verts[0])
        elif self.verts is not None:
            pc.update_mesh_properties(self.verts)

    # ---- host inputs -----------------------------------------------------------------------------------------------
    def _upload(self, dst, src_host):
        """H2D on the copy stream: after the last replay that read `dst`, concurrently with the main stream."""
        if self._done is not None:
            self._side.wait_event(self._done)
        with torch.cuda.stream(self._side):
            dst.copy_(src_host, non_blocking=True)
            self._gt_ready = torch.cuda.Event()
            self._gt_ready.record(self._side)

    def _await_upload(self):
        """The main stream waits for an upload in flight on the copy stream (before the replay that reads it)."""
        if self._gt_ready is not None:
            torch.cuda.current_stream(self.device).wait_event(self._gt_ready)
            self._gt_ready = None

    def _mark_read(self):
        """Records that the replays enqueued so far have read the uploaded buffers: the next upload waits for it."""
        self._done = torch.cuda.Event()
        self._done.record()

    # ---- capture ---------------------------------------------------------------------------------------------------
    def _learn_capacity(self):
        """Eager frames (sync modes EXACT then LATE) over the warm-up cameras, each at every warm-up timestep: their
        instance counts size the graph."""
        if self.K > 1:   # a K-view frame learns from K-view frames only (rasterizer.view_hints_of)
            hints, key = R.view_hints_of(self.pc), (self.device, self.W, self.H, self.pc._xyz.shape[0], self.K)
        else:
            hints, key = R.hints_of(self.pc), (self.device, self.W, self.H, self.pc._xyz.shape[0])
        n_max, lo, hi = 0, 0xFFFFFFFF, 0
        cam0 = self.cam.clone()
        pairs = self._warm_pairs
        t0 = self.timestep.clone() if self._warm_t or (pairs and self.timestep is not None) else None
        blocks = self._warm if self._warm else [cam0]
        steps = self._warm_t if self._warm_t else [None]
        runs = pairs if pairs else [(blk, t) for blk in blocks for t in steps]
        # eager frames on a side stream (torch's recipe for whole-step capture): nothing autograd creates here may be
        # tied to the legacy default stream
        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for rep in range(2):
                for blk, t in runs:
                    self.cam.copy_(blk)
                    if t is not None:
                        self.timestep.fill_(t)
                    self._body()
                    n_max = max(n_max, int((hints.last or {}).get("num_rendered", 0)))
                    d = hints.get(key)[1]
                    if d[1] > d[0]:  # union of the (already widened) depth-key ranges: one bucket grid fits all
                        lo, hi = min(lo, d[0]), max(hi, d[1])
        cur.wait_stream(side)
        # the frame's own camera and timestep again: the captured frame must not render the last warm-up one
        self.cam.copy_(cam0)
        if t0 is not None:
            self.timestep.copy_(t0)
        torch.cuda.synchronize(self.device)
        self._release()
        return n_max, ((lo, hi) if hi > lo else (0, 0))

    def _room_for(self, n: int) -> int:
        """The instance capacity of a graph whose frames need n instances."""
        return int(n * self.headroom) + 16384

    def capture(self, capacity: Optional[int] = None):
        self.graph = None
        self._before_capture()
        n_max, depth = self._learn_capacity()
        if capacity is None:
            capacity = self._capacity if self._capacity else self._room_for(n_max)
        self.slot = R.CaptureSlot(self.device, capacity, depth)
        self.graph = torch.cuda.CUDAGraph()
        R._capture_slot = self.slot
        try:
            with torch.cuda.graph(self.graph):
                self._body(captured=True)
        finally:
            R._capture_slot = None
        self._after_capture()
        self._key = self._state_key()
        self.captures += 1
        return self

    def _state_key(self):
        """What a capture baked in that eager code between replays may replace: P, active_sh_degree, the addresses
        of the binding and of the parameters and, with a FLAME head, the FLAME tensors' addresses and shapes and the
        in-place versions of shape / static_offset.  The timestep is read on the device and is not part of it."""
        pc = self.pc
        b = getattr(pc, "binding", None)
        key = [int(pc._xyz.shape[0]), int(getattr(pc, "active_sh_degree", 0)), None if b is None else b.data_ptr()]
        key += [p.data_ptr() for p in pc.parameters()]
        if self.flame is not None:
            for k in _FLAME_KEYS:
                t = pc.flame_param.get(k)
                key.append(None if t is None else (t.data_ptr(), tuple(t.shape)) +
                           ((t._version,) if k in ("shape", "static_offset") else ()))
        return key

    def _stale(self) -> bool:
        """No graph yet, or the model no longer matches what the capture baked in (host-side compare: no sync).  A
        frame whose key is None never re-captures."""
        return self.graph is None or (self._key is not None and self._state_key() != self._key)

    def _check_store(self, store):
        from .frames import FrameStore
        if not isinstance(store, FrameStore):
            raise ValueError(f"frames must be a gaussianavatars_b200.FrameStore, got {type(store).__name__}")
        if (store.W, store.H) != (self.W, self.H):
            raise ValueError(f"the frame store holds {store.W}x{store.H} frames, this frame renders {self.W}x{self.H}")
        if store.device != self.device:
            raise ValueError(f"the frame store lives on {store.device}, this frame on {self.device}")
        if not torch.equal(store.bg, self.bg):
            raise ValueError(f"the frame store's frames are composited over {store.bg.tolist()}, this frame renders "
                             f"over {self.bg.tolist()}: the backgrounds must be equal")
        if len(store) == 0:
            raise ValueError("the frame store holds no frames: add them before building the frame")

    # ---- a device-resident view schedule (schedule.ViewSchedule) ---------------------------------------------------
    def _use_schedule(self, schedule, store, log: bool):
        """Checks `schedule` against this frame and creates what the frame owns to follow it: the device `cursor`
        (the iteration the next replay runs), the `exhausted` word the sampler raises past the end of the order and,
        with log, the `losses` log ((L,) float32, NaN until its iteration commits).  Without warm cameras, the warm-up
        renders up to 16 records spread over the table, each at its own timestep."""
        from .schedule import ViewSchedule
        if not isinstance(schedule, ViewSchedule):
            raise ValueError(f"schedule must be a gaussianavatars_b200.ViewSchedule, got {type(schedule).__name__}")
        schedule.check_for(type(self).__name__, self.W, self.H, self.K, self.device,
                           self.num_timesteps if self.flame is not None else None, store)
        if self.flame is None and self.verts is not None:
            raise ValueError("this model is posed by host vertices: a schedule poses the model from its timesteps, "
                             "which needs a FLAME head (pc.flame), or a model without a mesh")
        self.schedule = schedule
        dev = self.device
        self.cursor = torch.zeros(1, dtype=torch.int32, device=dev)
        self.exhausted = torch.zeros(1, dtype=torch.int32, device=dev)
        self.losses = torch.full((schedule.L,), float("nan"), dtype=torch.float32, device=dev) if log else None
        self._cursor_host = self._pending = 0   # the cursor last read on the host, replays enqueued since
        if self._warm is None:
            ts = schedule.timesteps_host
            self._warm_pairs = [(schedule.cams[r] if self.K > 1 else schedule.cams[r, 0], None if ts is None else ts[r])
                                for r in schedule.warm_records()]

    def set_cursor(self, i: int):
        """The next replay runs iteration i of the schedule (resuming from a checkpoint; 0 rewinds).  Enqueued behind
        the replays so far; clears the exhausted word."""
        if self.schedule is None:
            raise ValueError("set_cursor needs a frame built with schedule=")
        i = int(i)
        if not 0 <= i <= self.schedule.L:
            raise IndexError(f"the cursor lies in [0, {self.schedule.L}], got {i}")
        self.cursor.fill_(i)
        self.exhausted.zero_()
        self._cursor_host, self._pending = i, 0

    def _launch_sample(self, ids=None, rows=None):
        """gab200_schedule_sample: record order[cursor] -> the camera block, the timestep, `ids`, `rows`."""
        s = self.schedule
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        t_out = self.timestep if s.timesteps is not None else None
        N.check(N.lib().gab200_schedule_sample(s.R, s.K, s.L, s.cams.data_ptr(), N.ptr(s.timesteps),
                                               N.ptr(s.frame_ids), s.order.data_ptr(), self.cursor.data_ptr(),
                                               self.cam.data_ptr(), N.ptr(t_out), N.ptr(ids), N.ptr(rows),
                                               self.exhausted.data_ptr(), stream), "gab200_schedule_sample")

    def _launch_commit(self, loss=None):
        """gab200_schedule_commit: unless this replay overflowed (the slot's sticky flag) or found the schedule
        exhausted, log `loss` at the cursor and advance it."""
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        N.check(N.lib().gab200_schedule_commit(self.schedule.L, self.slot.flag.data_ptr(), self.exhausted.data_ptr(),
                                               N.ptr(loss if self.losses is not None else None), N.ptr(self.losses),
                                               self.cursor.data_ptr(), stream), "gab200_schedule_commit")

    def _run_scheduled(self, n: int, check: bool):
        """n replays of the schedule's next iterations.  Refused on the host when they could run past the end of the
        order (the cursor last read plus the replays enqueued since: no sync).  check: one synchronisation, then the
        cursor and the overflow flag; after an overflow, regrow() and replay the iterations that did not commit.
        Returns the iterations committed since the cursor was last read (check=True), else None."""
        if self.schedule is None:
            raise ValueError("a scheduled run needs a frame built with schedule=")
        n, L = int(n), self.schedule.L
        if n < 0:
            raise ValueError(f"the number of iterations must be >= 0, got {n}")
        if self._cursor_host + self._pending + n > L:
            raise ValueError(f"{n} more iterations could run past the schedule's {L}: the cursor reaches up to "
                             f"{self._cursor_host + self._pending} (set_cursor rewinds)")
        if self._stale():
            self.capture()
        for _ in range(n):
            self._replay_scheduled()
        self._pending += n
        if not check:
            return None
        start, want, grown_at = self._cursor_host, self._cursor_host + self._pending, None
        while True:
            over = self.overflowed(wait=True)   # waits for the replays; then the cursor is a plain read
            c = int(self.cursor.item())
            if c == want:
                break
            if not over:
                raise RuntimeError(f"{type(self).__name__}: the schedule's cursor stopped at {c} of {want} without an "
                                   "overflow (exhausted: the cursor was moved past the order)")
            if grown_at == c:
                raise RuntimeError(f"{type(self).__name__}: iteration {c} still overflows its instance capacity after "
                                   "re-capture")
            grown_at = c
            self.regrow(c)   # an overflowed replay and the ones behind it committed nothing: redo them from c
            for _ in range(want - c):
                self._replay_scheduled()
        self._cursor_host, self._pending = want, 0
        return want - start

    # ---- overflow --------------------------------------------------------------------------------------------------
    def overflowed(self, wait: bool = True) -> bool:
        """True if any replay since the last (re-)capture needed more than the captured capacity.  The sticky flag stays
        on the device (a copy of it inside the graph would be the last node of every replay): wait=True reads it behind
        the replays enqueued so far; wait=False returns what the last wait=True read found."""
        if self.slot is None:
            return False
        if wait:
            torch.cuda.current_stream(self.device).synchronize()
            self.slot.flag_host.copy_(self.slot.flag)
        return bool(int(self.slot.flag_host[0]) != 0)

    def counters(self) -> dict:
        """Frame counters of the most recent finished replay (host copy; synchronise first for an exact answer)."""
        c = self.slot.counters
        return dict(num_rendered=int(c[R.N.CTR_NUM_RENDERED]) & 0xFFFFFFFF, capacity=int(c[R.N.CTR_CAPACITY]) & 0xFFFFFFFF,
                    bucket_overflow=int(c[R.N.CTR_BUCKET_OVERFLOW]), listed=int(c[R.N.CTR_NUM_LISTED]) & 0xFFFFFFFF)

    def regrow(self, iteration: Optional[int] = None):
        """Re-capture with the capacity the overflowing frame asked for (x headroom) and a fresh depth range.
        iteration: with a schedule whose records size the warm-up (no warm cameras), the iteration whose replay
        overflowed: its record joins the warm-up frames, so that the new depth range and capacity cover it too (a
        record at a timestep no warm-up frame posed can reach depths outside their range)."""
        torch.cuda.synchronize(self.device)
        if iteration is not None and self.schedule is not None and self._warm_pairs is not None:
            s, r = self.schedule, self.schedule.record(int(iteration))
            self._warm_pairs.append((s.cams[r] if self.K > 1 else s.cams[r, 0],
                                     None if s.timesteps_host is None else s.timesteps_host[r]))
        need = self.counters()["num_rendered"]
        self.capture(capacity=max(self._room_for(need), int(self.slot.capacity * 1.5)))


class GraphedFrame(_Captured):
    def __init__(self, pc, width: int, height: int, fovx: float, fovy: float, bg: torch.Tensor, loss: str = "l1_u8",
                 lambda_dssim: float = 0.2, host_inputs: bool = False, capacity: Optional[int] = None,
                 headroom: float = 1.25, after_backward=None, warm_cameras=None, regularizers: Optional[dict] = None,
                 before_backward=None, side_work=None, side_work_at: str = "start", optimizer: Optional[Adam] = None,
                 densify_stats: bool = False, per_camera_fov: bool = False, views_per_replay: int = 1,
                 rgba: bool = False, lambda_mask: float = 0.0, frames=None, schedule=None):
        """loss: "l1_u8" (L1 vs a uint8 ground truth), "photometric" ((1-l) L1 + l (1-SSIM) vs a uint8 ground truth) or
        "dL_dimage" (the caller supplies dL/dimage in `self.dL_dimage`).
        host_inputs: the frame owns pinned STAGING tensors (`cam_stage` (35,) float32, `gt_stage` (3,H,W) uint8) that a
        loader fills, and the graph ends with a D2H copy of the loss to `loss_host`.  How the staged inputs reach the
        device: (a) `set_inputs()` with HOST tensors uploads them on this frame's copy stream and `run()` makes the
        replay wait for them on the GPU; or (b) two frames used alternately prefetch for each other INSIDE their graphs
        (`a.prefetch_for(b); b.prefetch_for(a)` before capture): a forked branch of a's graph copies b's staging
        tensors into b's device buffers while a computes, so the upload of step i+1 runs under step i with no event
        between graphs.  (An H2D node at the HEAD of the consuming graph is what does not work: a 140-byte camera copy
        queues on the copy engine behind the 6 MB ground truth of the next step and delays every replay by that
        whole transfer; ordering uploads against replays with cross-stream events costs time every step as well.)
        after_backward: optional callable run inside the capture after backward (e.g. the gradient all-reduce).
        before_backward: the same, right before backward (e.g. attach this frame's gradient buffer to the model).
        side_work: optional callable captured on a FORKED branch of the graph that runs concurrently with the whole
        frame and is joined at its end -- e.g. the all-reduce of the PREVIOUS step's gradient buffer
        (dist.SymmetricGradBuffer.reduce of the other frame of an alternating pair), which then costs no step time.
        warm_cameras: camera blocks (35,) -- (37,) or camera objects with per_camera_fov -- rendered eagerly before the
        capture to size the instance capacity.
        regularizers: keyword arguments of `binding_regularizers` (threshold_xyz, lambda_scale, ...; {} = the
        reference's defaults): the position / scale terms of train.py:134-146 are added to the loss inside the graph.
        densify_stats: after backward (and after_backward) the graph accumulates the densification statistics of the
        frame into pc.xyz_gradient_accum / denom / max_radii2D (densify.add_densification_stats).
        optimizer: a capturable `Adam` (capturable=True) over the model's parameters; the graph ends with its step(),
        so one replay is one training iteration.  Capture leaves the parameters, moments, steps and statistics as
        they are: the first run() is the first step.  The frame remembers what the capture baked in (P,
        active_sh_degree, the addresses of every parameter, moment, step, statistic and binding, every group's
        hyper-parameters) and run() re-captures (`captures` counts it) when any of it changed: after
        densify_and_prune, reset_opacity or oneupSHdegree.  A learning rate written into a group on the host every
        iteration therefore re-captures every iteration: give the group an `lr_schedule` instead.  Not combinable
        with pair_with_deferred_reduce; a synchronous all-reduce in after_backward runs before the step.
        per_camera_fov: False (default): every replay renders with the fovx / fovy given here, baked into the graph --
        correct only for cameras that share that FoV.  True: the camera block is 37 floats, the last two
        tan(FoVx/2), tan(FoVy/2) (`camera_block(cam, fov=True)`), read by the kernels on every replay; fovx / fovy
        only seed the initial block.  set_inputs(camera=), warm_cameras, the staging tensors and prefetch_for then
        all carry 37 floats, and the warm-up sizes the capacity with each warm camera's own FoV.  The FoV is not
        part of what triggers a re-capture.
        views_per_replay=K > 1: one replay is one training iteration over K cameras of one timestep
        (renderer.render_views_train: one forward and one backward for the K views, the gradients summed over them).
        The camera input is a (K, 37) device table (per_camera_fov is implied): set_inputs(cameras=K camera objects
        of one image size, or a (K, 37) table), warm_cameras is a list of such groups, and gt_u8 / dL_dimage /
        gt_stage / image are (K,3,H,W), cam_stage (K,37), radii (K,P), viewspace_points (K,P,3).  The loss is
        K x the batch loss (one mean over the K images), i.e. the sum of the K per-view losses, plus the regularisers
        once per view with that view's radii; densify_stats feeds the K rows to the statistics in view order; the
        optimizer takes ONE step per replay.  Changing cameras, timestep or ground truth never re-captures.
        views_per_replay=1 is the single-camera frame.
        rgba=True: the ground truth arrives as the capture's decoded RGBA frame(s) -- `set_inputs(gt_rgba=...)`, uint8
        (H,W,4) or (K,H,W,4), in place of gt_u8, which is refused -- and the graph makes the (3,H,W) / (K,3,H,W) uint8
        ground truth itself before the loss: the reference loader's composite onto `bg`, bit for bit
        (training.composite_rgba).  `gt` holds the composite, `mask` the alpha bytes ((1,H,W) / (K,1,H,W)); gt_stage
        is the pinned (H,W,4) / (K,H,W,4) RGBA frame.  A loader then only decodes the PNG.
        lambda_mask > 0 (needs rgba=True): the frame renders the alpha plane as well (render(depth_alpha=True)),
        exposes `alpha` and `depth`, and adds the foreground-mask term  K * lambda_mask * l1_loss_u8(alpha, mask),
        the sum over the views of lambda_mask * mean|alpha - mask/255|, to the loss before the regularisers.  Both
        are construction constants: they never re-capture.
        frames=store (a frames.FrameStore of this frame's size, composited over this frame's bg): the ground truth and
        the mask are decoded inside the graph, at the point where rgba=True composites them, from the store's frames
        that `set_inputs(frames=...)` names -- K ids (an int when K = 1), each checked on the host against len(store)
        and written to a device int32 table without a host wait.  gt_u8 / gt_rgba are refused; lambda_mask > 0 uses
        the store's mask.  Only the camera table, the timestep and the K ids travel from the host per iteration; with
        host_inputs the ids are staged in the pinned `frames_stage` ((K,) int32, written by stage_frames) and travel
        beside cam_stage.  Changing ids never re-captures; a store that grew (its arena or index moved) does.  Not
        combinable with rgba=True or loss='dL_dimage'.
        schedule=s (a schedule.ViewSchedule): every captured replay runs the next iteration of the schedule by itself.
        A sampler kernel at its head copies record order[cursor] -- the camera table, the timestep, the K frame ids --
        into the frame's inputs, and a commit kernel at its end (after the optimizer step) logs the detached loss in
        `losses[cursor]` and advances the device `cursor`, unless the replay overflowed its capacity.
        run_iterations(n) enqueues n replays with no host input; set_cursor(i) resumes; loss_history(a, b) reads the
        log.  The warm-up renders `warm_cameras` if given, else up to 16 records of the table at their own timesteps.
        per_camera_fov is implied.  Refused: host_inputs, prefetch_for, loss='dL_dimage', rgba=True, a model posed by
        host vertices, and set_inputs(camera=, cameras=, timestep=, frames=).  The cursor and the log survive a
        re-capture (densify_and_prune, reset_opacity, oneupSHdegree between runs); the schedule never re-captures."""
        if schedule is not None:
            if host_inputs:
                raise ValueError("schedule= samples the inputs on the device: host_inputs=True stages them on the host; "
                                 "use one of them")
            if loss == "dL_dimage":
                raise ValueError("schedule= trains on a scalar loss ('l1_u8' or 'photometric'): loss='dL_dimage' "
                                 "takes a host-written gradient")
            if rgba:
                raise ValueError("schedule= cannot feed rgba=True: nothing on the device holds the RGBA frames to "
                                 "composite; add them to a FrameStore and give frames=store")
        if frames is not None and rgba:
            raise ValueError("frames= decodes the ground truth from the frame store: rgba=True composites it from an "
                             "RGBA input instead; use one of them")
        if frames is not None and loss == "dL_dimage":
            raise ValueError("frames= decodes the ground truth of a scalar loss ('l1_u8' or 'photometric'): "
                             "loss='dL_dimage' reads none")
        if loss not in ("l1_u8", "photometric", "dL_dimage"):
            raise ValueError("loss must be 'l1_u8', 'photometric' or 'dL_dimage'")
        if regularizers is not None and loss == "dL_dimage":
            raise ValueError("regularizers need a scalar loss ('l1_u8' or 'photometric')")
        if rgba and loss == "dL_dimage":
            raise ValueError("rgba=True makes the ground truth of a scalar loss ('l1_u8' or 'photometric'): "
                             "loss='dL_dimage' reads none")
        lambda_mask = float(lambda_mask)
        if not lambda_mask >= 0.0 or not math.isfinite(lambda_mask):
            raise ValueError(f"lambda_mask must be a finite value >= 0, got {lambda_mask}")
        if lambda_mask > 0.0 and not rgba and frames is None:
            raise ValueError("the mask term compares the alpha plane with the capture's alpha: lambda_mask > 0 "
                             "needs rgba=True")
        if optimizer is not None and not (isinstance(optimizer, Adam) and
                                          all(g.get("capturable", False) for g in optimizer.param_groups)):
            raise ValueError("optimizer must be a gaussianavatars_b200.Adam with capturable=True")
        _check_views_per_replay(views_per_replay)
        self.K = int(views_per_replay)
        super().__init__(pc, width, height, fovx, fovy, bg, per_camera_fov or self.K > 1 or schedule is not None,
                         capacity, headroom, warm_cameras, verts_grad=True)
        self.loss_kind, self.lambda_dssim, self.host_inputs = loss, float(lambda_dssim), bool(host_inputs)
        self.after_backward = after_backward
        self.before_backward = before_backward   # e.g. SymmetricGradBuffer.begin
        self.side_work = side_work
        self.side_work_at = side_work_at   # "start": beside the whole frame; "backward": forked after the forward
        self.regularizers = regularizers
        self.optimizer = optimizer
        self.densify_stats = bool(densify_stats)
        self.rgba, self.lambda_mask = bool(rgba), lambda_mask
        self.frames = frames
        dev = self.device
        if frames is not None:
            self._check_store(frames)
        img = self._gt_shape()
        self.gt = torch.zeros(img, dtype=torch.uint8, device=dev) if loss != "dL_dimage" else None
        lead = () if self.K == 1 else (self.K,)
        # rgba: the static RGBA input the composite reads, and the mask it writes beside gt
        self.gt_rgba = torch.zeros(lead + (self.H, self.W, 4), dtype=torch.uint8, device=dev) if self.rgba else None
        self.mask = (torch.zeros(lead + (1, self.H, self.W), dtype=torch.uint8, device=dev)
                     if self.rgba or frames is not None else None)
        # frames: the device table of the K frame ids the decode reads (id 0 until set_inputs names others)
        self.frame_ids = torch.zeros(self.K, dtype=torch.int32, device=dev) if frames is not None else None
        self.frames_stage = (torch.zeros(self.K, dtype=torch.int32).pin_memory()
                             if frames is not None and host_inputs else None)
        gt_in = self._gt_input()
        self.dL_dimage = torch.zeros(img, dtype=torch.float32, device=dev) if loss == "dL_dimage" else None
        self.cam_host = torch.zeros(self.cam.shape, dtype=torch.float32).pin_memory() if host_inputs else None  # staging
        if self.cam_host is not None:
            self.cam_host.copy_(self.cam)
        self.cam_stage = self.cam_host
        self.gt_stage = (torch.zeros(gt_in.shape, dtype=torch.uint8).pin_memory()
                         if host_inputs and gt_in is not None else None)
        self._prefetch_target = None
        self.loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
        self.loss = None
        self.image = self.radii = self.viewspace_points = self.alpha = self.depth = None
        self._side = torch.cuda.Stream(device=dev) if (host_inputs or side_work is not None) else None
        self._uploads = bool(host_inputs)
        if schedule is not None:
            self._use_schedule(schedule, frames, log=True)

    def _gt_input(self):
        """The device tensor the ground truth is written into: the RGBA frame(s) with rgba=True, else gt; None with a
        frame store (the graph decodes gt itself)."""
        if self.frames is not None:
            return None
        return self.gt_rgba if self.rgba else self.gt

    def _frame_list(self, frames) -> list:
        """set_inputs' / stage_frames' ids: K ints (an int when K = 1), each checked against len(store)."""
        if self.frames is None:
            raise ValueError("frames= needs a GraphedFrame built with frames=store")
        if isinstance(frames, int) and not isinstance(frames, bool) and self.K > 1:
            raise ValueError(f"this frame trains {self.K} views per replay: give {self.K} frame ids")
        ids = self.frames.check_ids(frames)
        if len(ids) != self.K:
            raise ValueError(f"this frame trains {self.K} views per replay, got {len(ids)} frame ids")
        return ids

    def stage_frames(self, frames):
        """host_inputs: checks the ids and writes them into the pinned `frames_stage`, which the other frame of a
        prefetching pair copies in its graph (or upload_staged).  The caller keeps the stage as it keeps cam_stage:
        not rewritten while a replay that copies it may be running."""
        if self.frames_stage is None:
            raise ValueError("stage_frames needs a frame built with frames=store and host_inputs=True")
        self.frames_stage.copy_(torch.tensor(self._frame_list(frames), dtype=torch.int32))

    # ---- inputs ------------------------------------------------------------------------------------------------
    def set_inputs(self, camera=None, verts=None, gt_u8=None, dL_dimage=None, timestep=None, cameras=None,
                   gt_rgba=None, frames=None):
        """Copies new inputs into the static buffers (device tensors) / staging buffers (host_inputs).  `timestep`
        (a model with a FLAME head only) is a host int checked against the model's number of timesteps.
        views_per_replay=K > 1: `cameras` (K camera objects of the frame's image size, or a (K, 37) table) instead of
        `camera`; gt_u8 / dL_dimage are (K,3,H,W).  rgba=True: `gt_rgba`, the decoded uint8 RGBA frame (H,W,4) or
        (K,H,W,4), instead of gt_u8.  frames=store: `frames`, the K frame ids to decode (an int when K = 1)."""
        if self.schedule is not None and any(x is not None for x in (camera, cameras, timestep, frames)):
            raise ValueError("this frame samples its camera, timestep and frame ids from its schedule on the device: "
                             "set_inputs(camera=, cameras=, timestep=, frames=) is refused (set_cursor moves it)")
        if (camera is not None and self.K > 1) or (cameras is not None and self.K == 1):
            raise ValueError("a frame with views_per_replay > 1 takes cameras=, one with a single view camera=")
        if (gt_u8 is not None or gt_rgba is not None) and self.frames is not None:
            raise ValueError("this frame decodes its ground truth from the frame store: give frames=, not gt_u8 / "
                             "gt_rgba")
        ids = self._frame_list(frames) if frames is not None else None
        if gt_u8 is not None and self.rgba:
            raise ValueError("this frame composites its ground truth from the RGBA frame: give gt_rgba=, not gt_u8")
        if gt_rgba is not None:
            if not self.rgba:
                raise ValueError("gt_rgba= needs a frame built with rgba=True")
            if gt_rgba.dtype != torch.uint8 or tuple(gt_rgba.shape) != tuple(self.gt_rgba.shape):
                raise ValueError(f"gt_rgba of this frame is a uint8 {tuple(self.gt_rgba.shape)} tensor, got "
                                 f"{gt_rgba.dtype} {tuple(gt_rgba.shape)}")
        if cameras is not None:
            camera = cameras
        for name, t in (("gt_u8", gt_u8), ("dL_dimage", dL_dimage)):
            if t is not None and self.K > 1 and tuple(t.shape) != self._gt_shape():
                raise ValueError(f"{name} of this frame is {self._gt_shape()}, got {tuple(t.shape)}")
        if camera is not None and self.K > 1 and not isinstance(camera, torch.Tensor):
            sizes = {(int(c.image_width), int(c.image_height)) for c in camera}
            if sizes != {(self.W, self.H)}:
                raise ValueError(f"the cameras of this frame are {self.W}x{self.H}, got {sorted(sizes)}")
        self._set_pose_input(verts, timestep)
        if camera is not None:
            blk = self._camera_tensor(camera)
            if blk.device.type == "cpu" and self._uploads:
                if not blk.is_pinned():      # stage pageable memory (after any upload still reading the staging copy)
                    self._side.synchronize()
                    self.cam_host.copy_(blk)
                    blk = self.cam_host
                self._upload(self.cam, blk)
            else:
                self.cam.copy_(blk, non_blocking=True)
        if verts is not None:
            with torch.no_grad():
                self.verts.copy_(verts.reshape(self.verts.shape), non_blocking=True)
        gt_src = gt_rgba if gt_rgba is not None else gt_u8
        if gt_src is not None:
            dst = self._gt_input()
            if gt_src.device.type == "cpu" and self._uploads:
                self._upload(dst, gt_src)
            else:
                dst.copy_(gt_src, non_blocking=True)
        if dL_dimage is not None:
            self.dL_dimage.copy_(dL_dimage, non_blocking=True)
        if ids is not None:
            if self._uploads:   # through the pinned stage, on the copy stream, like a host camera
                self._side.synchronize()
                self.stage_frames(ids)
                self._upload(self.frame_ids, self.frames_stage)
            elif self.K == 1:   # a fill, like the timestep
                self.frame_ids.fill_(ids[0])
            else:   # a pinned block of the caching allocator: the copy does not wait on the host
                self.frame_ids.copy_(torch.tensor(ids, dtype=torch.int32).pin_memory(), non_blocking=True)

    def prefetch_for(self, other: "GraphedFrame"):
        """This frame's graph will, on a forked branch, copy `other`'s pinned staging tensors (cam_stage, gt_stage)
        into `other`'s device inputs while it computes.  Call before capture()."""
        if getattr(self, "schedule", None) is not None or getattr(other, "schedule", None) is not None:
            raise ValueError("a frame with schedule= takes no host inputs: it cannot join a prefetching pair")
        if not (self.host_inputs and other.host_inputs):
            raise ValueError("prefetching needs host_inputs=True on both frames")
        if self.per_camera_fov != other.per_camera_fov:
            raise ValueError("both frames of a prefetching pair must use the same per_camera_fov mode")
        if self.K != other.K:
            raise ValueError("both frames of a prefetching pair must render the same number of views per replay")
        if self.rgba != other.rgba:
            raise ValueError("both frames of a prefetching pair must take the same ground truth (rgba=True on both "
                             "or on neither)")
        if (self.frames is None) != (other.frames is None):
            raise ValueError("both frames of a prefetching pair must take the same ground truth (frames= on both or "
                             "on neither)")
        self._prefetch_target = other
        return self

    def upload_staged(self):
        """Eager upload of this frame's own staging tensors (the first step of a prefetching pair)."""
        self.cam.copy_(self.cam_stage, non_blocking=True)
        if self.gt_stage is not None:
            self._gt_input().copy_(self.gt_stage, non_blocking=True)
        if self.frames_stage is not None:
            self.frame_ids.copy_(self.frames_stage, non_blocking=True)

    # ---- the step body (run eagerly for warm-up, then captured) --------------------------------------------------
    def _params(self):
        """The tensors whose gradients the graph produces: the splat parameters, then the trained FLAME tensors."""
        ps = list(self.pc.parameters())
        if self.flame is not None:
            ps += [self.pc.flame_param[k] for k in _FLAME_KEYS[2:] if self.pc.flame_param[k].requires_grad]
        return ps

    def _body(self, captured: bool = False):
        """One frame; `captured` (the graph, not the warm-up frames) also accumulates the statistics and steps the
        optimizer."""
        pc = self.pc
        for p in self._params():
            p.grad = None
        if self.verts is not None:
            self.verts.grad = None
        if captured and self.schedule is not None:   # this replay's record: camera table, timestep, frame ids
            self._launch_sample(ids=self.frame_ids)
        other = self._prefetch_target
        forked = other is not None or self.side_work is not None
        if forked:   # forked branch: runs while this frame computes
            cur = torch.cuda.current_stream(self.device)
            self._side.wait_stream(cur)
            with torch.cuda.stream(self._side):
                if other is not None:   # the other frame's next inputs travel
                    other.cam.copy_(other.cam_stage, non_blocking=True)
                    if other.gt_stage is not None:
                        other._gt_input().copy_(other.gt_stage, non_blocking=True)
                    if other.frames_stage is not None:
                        other.frame_ids.copy_(other.frames_stage, non_blocking=True)
                if self.side_work is not None and self.side_work_at == "start":
                    self.side_work()
        self._pose()
        planes = self.lambda_mask > 0.0   # the mask term reads the alpha plane
        if self.K > 1:   # the K cameras of the table in one forward and one backward
            out = render_views_train(self.cam, pc, _Pipe, self.bg, width=self.W, height=self.H, depth_alpha=planes)
        else:
            out = render(self.camera, pc, _Pipe, self.bg, depth_alpha=planes)
        img = out["render"]
        radii_rows = [out["radii"]] if self.K == 1 else list(out["radii"])
        if self.rgba:   # the loader's composite of the RGBA input: gt and mask for this replay's loss
            launch_composite_rgba(self.gt_rgba, self.bg, self.gt, self.mask)
        elif self.frames is not None:   # the same gt and mask, decoded from the store's frames of the device ids
            self.frames.launch_decode(self.frame_ids, self.gt, self.mask)
        if self.loss_kind in ("l1_u8", "photometric"):
            loss = l1_loss_u8(img, self.gt) if self.loss_kind == "l1_u8" else photometric_loss(img, self.gt, self.lambda_dssim)
            if self.K > 1:   # one mean over the K images: K x it is the sum of the per-view losses
                loss = loss * float(self.K)
            if planes:   # one mean over the K alpha planes, K x it: the sum of the per-view mask terms
                loss = loss + l1_loss_u8(out["alpha"], self.mask) * (float(self.K) * self.lambda_mask)
            if self.regularizers is not None:
                for radii in radii_rows:   # train.py:134-146 per view, with that view's visibility
                    lx, ls = binding_regularizers(pc._xyz, pc._scaling, radii, getattr(pc, "binding", None),
                                                  getattr(pc, "face_scaling", None), **self.regularizers)
                    loss = loss + lx + ls
            self._fork_side_at_backward()
            if self.before_backward is not None:
                self.before_backward()
            loss.backward()
        else:
            loss = None
            self._fork_side_at_backward()
            if self.before_backward is not None:
                self.before_backward()
            img.backward(self.dL_dimage)
        if self.after_backward is not None:
            self.after_backward()
        if captured:
            skip = self.slot.flag
            if self.densify_stats:
                if self.K == 1:
                    add_densification_stats(pc, out["viewspace_points"], out["radii"], skip_flag=skip)
                else:   # the K views' rows in view order: the state after K single-view frames
                    vp = out["viewspace_points"].grad
                    for k in range(self.K):
                        add_densification_stats(pc, SimpleNamespace(grad=vp[k]), out["radii"][k], skip_flag=skip)
            if self.optimizer is not None:
                self.optimizer.step(skip_flag=skip)
        if loss is not None:
            self.loss = loss.detach()
            self.loss_host.copy_(self.loss, non_blocking=True)
        if forked:   # join the branch (a captured fork must end inside the graph)
            torch.cuda.current_stream(self.device).wait_stream(self._side)
        if captured and self.schedule is not None:   # log the loss and advance the cursor, unless this replay overflowed
            self._launch_commit(self.loss)
        self.image, self.radii, self.viewspace_points = img.detach(), out["radii"], out["viewspace_points"]
        if planes:
            self.alpha, self.depth = out["alpha"].detach(), out["depth"].detach()

    def _fork_side_at_backward(self):
        if self.side_work is not None and self.side_work_at == "backward":
            self._side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self._side):
                self.side_work()

    # ---- capture ---------------------------------------------------------------------------------------------------
    def _release(self):
        """What the warm-up frames left on the model / on this object: tensors with autograd history."""
        self.pc.face_center = self.pc.face_orien_mat = self.pc.face_scaling = None
        if self.flame is not None:
            self.pc.verts_cano = None
        self.image = self.radii = self.viewspace_points = self.loss = self.alpha = self.depth = None

    def _before_capture(self):
        if self.optimizer is not None:
            self.optimizer.init_state()   # created inside the capture, the state would be re-zeroed by every replay

    def _after_capture(self):
        # the tensors autograd left in .grad during the capture ARE the graph's outputs: remember them, a second
        # GraphedFrame of the same model re-points .grad at its own when it captures
        self.grads = [p.grad for p in self._params()]
        self.flat_grad = getattr(self.pc, "flat_grad", None)

    def _state_key(self):
        """Everything a training capture baked in that eager code between replays may replace: beyond the shared key,
        which FLAME tensors receive gradients, the statistics, every group's hyper-parameters and the addresses of
        every moment and step, and with a frame store the addresses of its arena and index.  None for a frame that
        neither trains, poses a FLAME head nor reads a store: it never re-captures."""
        pc = self.pc
        if self.optimizer is None and not self.densify_stats and self.flame is None and self.frames is None:
            return None
        key = super()._state_key()
        if self.frames is not None:
            key.append(self.frames.pointers())
        if self.flame is not None:
            key += [t is not None and t.requires_grad for t in map(pc.flame_param.get, _FLAME_KEYS)]
        if self.densify_stats:
            key += [getattr(pc, n).data_ptr() for n in _STATS]
        opt = self.optimizer
        if opt is not None:
            for g in opt.param_groups:
                sched = g.get("lr_schedule")
                key.append((tuple(sorted(sched.items())) if sched is not None else float(g["lr"]),
                            tuple(g["betas"]), float(g["eps"])))
                for p in g["params"]:
                    st = opt.state.get(p, {})
                    key.append((p.data_ptr(), p.shape) + tuple(st[k].data_ptr() for k in ("step", "exp_avg", "exp_avg_sq")
                                                               if k in st))
        return key

    # ---- replay ----------------------------------------------------------------------------------------------------
    def run(self, check: bool = False):
        if self.schedule is not None:   # one iteration of the schedule
            self._run_scheduled(1, check)
            return self
        if self._stale():
            self.capture()
        self._await_upload()   # a ground-truth upload in flight on the copy stream
        self._replay()
        if self._uploads:
            self._mark_read()
        if check and self.overflowed(wait=True):
            self.regrow()
            self._replay()
            if self.overflowed(wait=True):
                raise RuntimeError("GraphedFrame: the frame still overflows its instance capacity after re-capture")
        return self

    def _replay(self):
        """One replay, counted, with .grad pointing at this graph's gradients again."""
        self.graph.replay()
        self.replays += 1
        for p, g in zip(self._params(), self.grads):
            p.grad = g
        self.pc.flat_grad = self.flat_grad

    _replay_scheduled = _replay

    def run_iterations(self, n: int, check: bool = True):
        """schedule=: n training iterations of the schedule as n back-to-back replays, with no host input between
        them (re-capturing first if the model changed).  Refused on the host, before anything runs, when they could
        pass the end of the order.  check=True synchronises once at the end and reads the cursor and the overflow
        flag: if a replay overflowed its capacity, it skipped its statistics, its Adam step and its commit, and so did
        every replay behind it in the run (the sticky flag) -- wasted work, not wrong work; the frame then regrows and
        replays from the record that overflowed.  Returns the number of iterations committed (n, when no unchecked
        run came before); check=False returns None and reads nothing."""
        return self._run_scheduled(n, check)

    def loss_history(self, a: int = 0, b: Optional[int] = None) -> torch.Tensor:
        """The logged losses of iterations a .. b - 1 of the schedule as a host tensor (one synchronisation); NaN for
        an iteration not committed yet."""
        if self.schedule is None:
            raise ValueError("loss_history needs a frame built with schedule=")
        return self.losses[a:b].cpu()


class GraphedRender(_Captured):
    """One PLAYBACK frame as ONE forward-only CUDA graph: what the reference's render.py, the fps benchmarks and the
    viewer run per frame (select_mesh_by_timestep(t) -> render() -> the uint8 frame), with no backward, no loss and
    no ground truth.

        view = GraphedRender(pc, width, height, bg, outputs="u8", host_slots=2)
        view.set_inputs(camera=cam, timestep=t)          # device buffers: never a re-capture
        view.run()                                       # enqueue one replay
        view.display, view.image, view.radii             # static result tensors ((H,W,3) uint8, (3,H,W) float32)

    What is captured: [the FLAME pose of the device timestep (pc.flame), or the given vertices in `verts`] -> the
    per-face frame (update_mesh_properties) -> the fused forward (need_backward = 0, GAB200_SYNC_NONE) writing the
    float image and/or the display image (gab200_forward_display: bit for bit render.py's
    mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(uint8)).  With mesh_update=False the graph renders the
    face frame the model holds (pc.face_center ...) at capture: eager update_mesh_properties calls replace those
    tensors and re-capture.

    The camera is always the 37-float block with the field of view (`camera_block(cam, fov=True)`: a viewer zooms);
    camera, timestep, vertices and background are device buffers written by `set_inputs`.  The parameters and the
    rows of pc.flame_param are read by address on every replay, so in-place edits (a viewer's FLAME sliders) show in
    the next one.  run() re-captures when the model, the image size or `scaling_modifier` changed (`captures` counts
    it): P, active_sh_degree, the addresses of the parameters and of the binding, the FLAME tensors' addresses and
    shapes and the in-place versions of shape / static_offset.

    The instance capacity is sized and guarded as in GraphedFrame: eager frames over `warm_cameras` (x `headroom`),
    a sticky overflow flag, `run(check=True)` re-captures with room and replays, `overflowed()`, `regrow()`.  The
    graph owns its scratch (allocated during the capture, in the graph's private pool), so eager no_grad renders,
    whose pooled scratch grows and moves, never touch it.

    host_slots=k > 0: after each replay the display frame travels to a ring of k pinned host tensors on a copy
    stream, one event per replay, so the copy of frame i overlaps replay i+1 (a consumer one replay behind never
    waits for a transfer).  `host_frame(i)` waits for replay i's copy and returns its slot; slot i % k is rewritten
    by replay i + k, not before.

    mesh_opacity=o: the tracked mesh drawn over the avatar, as the reference's viewers do (train.py:82-93,
    local_viewer.py's "show mesh"): the graph renders the float splat image, then the mesh overlay kernels
    (mesh.mesh_overlay) composite the mesh of the vertices the graph just posed at opacity o and write `display`.
    Pixels the mesh does not reach get the bytes the display epilogue would have written.  Opacity and face_colors
    ((F,3), e.g. the viewer's splats-per-face colouring) are device buffers written by set_inputs: a slider or a colour
    picker never re-captures.  `mesh_error` is a device int32 set to 1 when a face index is out of range.  With
    views_per_replay=K the mesh is drawn under all K cameras in one launch sequence (mesh.mesh_overlay_views), each
    view bit for bit its single-camera overlay.

    quantize="viewer": `display` holds the bytes the reference's local viewer exports (local_viewer.py's
    (np.clip(rgb, 0, 1) * 255).astype(np.uint8): a float32 multiply and truncation, no +0.5) instead of render.py's,
    written by the same blend epilogue -- or, with mesh_opacity, by the same mesh resolve -- with no extra pass.

    schedule=s (a schedule.ViewSchedule, e.g. trajectory.CameraPath.schedule()): every captured replay plays the next
    record of the schedule by itself.  A sampler kernel at its head copies record order[cursor] -- the camera row and
    the timestep -- into the frame's inputs, and a commit kernel at its end advances the device `cursor` unless the
    replay overflowed its capacity (csrc/schedule.cu, as GraphedFrame and GraphedEval use them).  run_all() plays the
    rest of the order, run_iterations(n) the next n records, set_cursor(i) moves the cursor; set_inputs(camera=,
    cameras=, timestep=) is refused.  With check=True one synchronisation ends the run; a replay that overflowed, and
    every replay behind it, committed nothing, so the frame regrows and replays from the record that overflowed."""

    _MESH_OVER_GT = False   # the mesh is drawn over the splat image into `display` (GraphedEval: over `gt`)

    def __init__(self, pc, width: int, height: int, bg: torch.Tensor, outputs: str = "u8",
                 scaling_modifier: float = 1.0, mesh_update: bool = True, host_slots: int = 0,
                 capacity: Optional[int] = None, headroom: float = 1.25, warm_cameras=None, warm_timesteps=None,
                 mesh_opacity: Optional[float] = None, face_colors: Optional[torch.Tensor] = None,
                 mesh_lighting: str = "front", views_per_replay: int = 1, depth_alpha: bool = False,
                 png: bool = False, quantize: str = "render", schedule=None):
        """outputs: "u8" (the display image only: the float image is not written), "float" or "both".
        warm_cameras: camera objects or 37-float blocks rendered eagerly before the capture to size the capacity (and
        the depth-sort range); warm_timesteps: with a FLAME head, the timesteps each warm camera is rendered at
        (default: the current one) -- a sequence played back whole sizes the graph once for all its frames.
        views_per_replay=K > 1: every replay renders K cameras of one timestep in one forward
        (gab200_forward_views): the head is posed once, set_inputs(cameras=...) takes K cameras (or a (K, 37) table),
        warm_cameras is a list of such camera groups, and display / image / radii / the host slots carry a leading K
        dimension; with mesh_opacity the mesh is drawn over each of the K float images into `display` (K,H,W,3).
        depth_alpha=True: every replay also refreshes `alpha` and `depth`, (1,H,W) float32 static tensors -- the
        splats' accumulated opacity and alpha-weighted view-space depth from the same blend (gab200_forward_depth_alpha;
        with the mesh overlay they remain the splats').  Single-view replays only.
        png=True: the captured body ends in the PNG encode of `display` (after the mesh overlay; png.encode_png's
        kernels) into graph-owned scratch, `png_out` ((K, capacity) uint8) and `png_len` ((K,) int64).  With
        host_slots the ring also receives the compressed files, and host_png(i) returns replay i's file (K files with
        views_per_replay=K).
        quantize: the bytes of `display`, "render" (render.py's, the default) or "viewer" (the local viewer's export);
        "viewer" needs outputs 'u8' or 'both' and is not combinable with depth_alpha.
        schedule: a ViewSchedule the replays follow on the device (see the class documentation)."""
        if outputs not in ("u8", "float", "both"):
            raise ValueError("outputs must be 'u8', 'float' or 'both'")
        N.quantize_mode(quantize)
        if quantize != "render" and (outputs == "float" or depth_alpha):
            raise ValueError("quantize='viewer' quantises the display image of a frame without the alpha / depth "
                             "planes: it needs outputs 'u8' or 'both' and depth_alpha=False")
        if png and outputs == "float":
            raise ValueError("png=True encodes the display image: it needs outputs 'u8' or 'both'")
        _check_views_per_replay(views_per_replay)
        if depth_alpha and views_per_replay > 1:
            raise ValueError("depth_alpha renders one camera per replay: it needs views_per_replay=1 (the K-view "
                             "forward has no alpha / depth planes)")
        self.K = int(views_per_replay)
        if host_slots < 0 or (host_slots > 0 and outputs == "float"):
            raise ValueError("host_slots copies the display image: it needs outputs 'u8' or 'both'")
        # the background is an input (set_inputs writes it): the frame's own copy.  Field of view: tan(45 deg), a
        # harmless one until the first camera arrives
        super().__init__(pc, width, height, math.pi / 2, math.pi / 2, bg.clone(), True, capacity, headroom,
                         warm_cameras, warm_timesteps)
        self.outputs, self.scaling_modifier, self.mesh_update = outputs, float(scaling_modifier), bool(mesh_update)
        self.host_slots = int(host_slots)
        self.png = bool(png)
        self.png_out = self.png_len = self._png_scratch = None
        self.host_png_slots = self._png_staged = None
        self.host = self._copy_stream = None
        self._staged = self._host_events = self._stage_events = None
        self.image = self.display = self.radii = self.alpha = self.depth = None
        self.depth_alpha = bool(depth_alpha)
        self.mesh = mesh_opacity is not None
        self.mesh_display = self.mesh_png_out = self.mesh_png_len = None
        self.host_mesh_png_slots = self._mesh_png_staged = None
        if self.mesh:
            if outputs == "float" and not self._MESH_OVER_GT:
                raise ValueError("the mesh overlay writes the display image: it needs outputs 'u8' or 'both'")
            if getattr(pc, "faces", None) is None:
                raise ValueError("mesh_opacity needs a model with a mesh (pc.faces)")
            if pc.faces.dtype not in (torch.int32, torch.int64):
                raise ValueError(f"the mesh overlay draws integer faces: pc.faces is {pc.faces.dtype}, not int32 / "
                                 "int64")
            if mesh_lighting not in M.LIGHTING:
                raise ValueError(f"mesh_lighting must be one of {sorted(M.LIGHTING)}, got {mesh_lighting!r}")
            self.mesh_lighting = mesh_lighting
            self._opacity = M.opacity_pair(mesh_opacity, self.device)
            self.face_colors = None
            if face_colors is not None:
                self._set_face_colors(face_colors)
            self.mesh_error = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._adjacency = M._AdjacencyCache()
        self.quantize = quantize
        if schedule is not None:
            self._use_schedule(schedule, None, log=False)

    def _set_face_colors(self, face_colors):
        fc = face_colors.detach().reshape(-1, 3)
        if fc.shape[0] != self.pc.faces.shape[0]:
            raise ValueError(f"face_colors must be (F,3) or (1,F,3) with F = {self.pc.faces.shape[0]}")
        if self.face_colors is None:   # a new buffer: the next run() re-captures (its address joins the state key)
            self.face_colors = fc.to(self.device, torch.float32).contiguous().clone()
        else:
            self.face_colors.copy_(fc, non_blocking=True)

    # ---- inputs ------------------------------------------------------------------------------------------------
    def set_inputs(self, camera=None, timestep=None, verts=None, bg=None, mesh_opacity=None, face_colors=None,
                   cameras=None):
        """Copies new inputs into the graph's device buffers; none of them re-captures.  A camera OBJECT of another
        image size changes the frame's size (the next run() re-captures).  views_per_replay=K > 1: `cameras` (K
        camera objects of one size, or a (K, 37) table) instead of `camera`."""
        if self.schedule is not None and any(x is not None for x in (camera, cameras, timestep)):
            raise ValueError("this frame samples its camera and timestep from its schedule on the device: "
                             "set_inputs(camera=, cameras=, timestep=) is refused (set_cursor moves it)")
        if (camera is not None and self.K > 1) or (cameras is not None and self.K == 1):
            raise ValueError("a frame with views_per_replay > 1 takes cameras=, one with a single view camera=")
        if cameras is not None:
            camera = cameras
        if (mesh_opacity is not None or face_colors is not None) and not self.mesh:
            raise ValueError("mesh_opacity / face_colors need a GraphedRender built with mesh_opacity=")
        if mesh_opacity is not None:
            self._opacity.copy_(M.opacity_pair(mesh_opacity, "cpu"), non_blocking=True)
        if face_colors is not None:
            self._set_face_colors(face_colors)
        self._set_pose_input(verts, timestep)
        if camera is not None:
            blk = self._camera_tensor(camera)
            if not isinstance(camera, torch.Tensor):
                first = camera if self.K == 1 else list(camera)[0]
                self.W, self.H = int(first.image_width), int(first.image_height)
                if self.camera is not None:
                    self.camera.image_width, self.camera.image_height = self.W, self.H
            self.cam.copy_(blk, non_blocking=True)
        if verts is not None:
            if self.verts is None:
                self.verts = verts.detach().reshape(-1, 3).to(self.device).float().contiguous().clone()
            else:
                self.verts.copy_(verts.detach().reshape(self.verts.shape), non_blocking=True)
        if bg is not None:
            self.bg.copy_(bg, non_blocking=True)

    # ---- the frame body (run eagerly for warm-up, then captured) -------------------------------------------------
    def _body(self, captured: bool = False):
        scheduled = captured and self.schedule is not None
        if scheduled:   # this replay's record: camera row and timestep
            self._launch_sample()
        self._frame(captured)
        if scheduled:   # advance the cursor, unless this replay overflowed
            self._launch_commit()

    def _frame(self, captured: bool):
        """The playback frame: pose, forward, mesh overlay, PNG encode."""
        with torch.no_grad():
            if self.mesh_update:
                self._pose()
            # K > 1: the K cameras of the table in one forward
            over = self.mesh and not self._MESH_OVER_GT   # the mesh over the float splat image(s)
            out = _forward_only(self.camera if self.K == 1 else self.cam, self.pc, _Pipe, self.bg,
                                self.scaling_modifier, self.outputs != "float" and not over,
                                self.outputs != "u8" or over, self.depth_alpha,
                                None if self.K == 1 else (self.W, self.H),
                                "render" if over else self.quantize)   # with the mesh, its resolve quantises
            if over:
                out["display_u8"] = self._overlay(out["render"])
        self.image, self.display, self.radii = out["render"], out["display_u8"], out["radii"]
        self.alpha, self.depth = out.get("alpha"), out.get("depth")
        if captured and self.png:   # the warm-up frames encode nothing
            self._encode_png()

    def _encode_png(self):
        """The display frame(s) -> PNG files in buffers the capture allocates (the graph's own pool)."""
        self._png_scratch = PNG.scratch(self.K, self.H, self.W, self.device)
        self.png_out, self.png_len = self._encode(self.display)

    def _encode(self, u8):
        """u8 (H,W,3) | (K,H,W,3) -> (files (K, stride) uint8, lengths (K,) int64), through the frame's PNG scratch."""
        K, dev = self.K, self.device
        out = torch.empty((K, PNG.slot_stride(self.W, self.H)), dtype=torch.uint8, device=dev)
        length = torch.empty(K, dtype=torch.int64, device=dev)
        PNG.launch_encode(u8, self._png_scratch, out, length)
        return out, length

    def _overlay(self, base):
        """The mesh of the vertices the frame just posed (pc.verts) over `base` -- the float splat image(s), or the
        uint8 ground truth -- at the frame's camera(s) -> (H,W,3) uint8, or (K,H,W,3) in one K-view call."""
        pc = self.pc
        if pc.verts is None:
            raise ValueError("the mesh overlay draws the posed vertices (pc.verts): pose the model first")
        faces = getattr(pc, "faces_i32", None)
        faces = pc.faces.to(torch.int32).contiguous() if faces is None else faces
        shape = (self.H, self.W, 3) if self.K == 1 else (self.K, self.H, self.W, 3)
        display = torch.empty(shape, dtype=torch.uint8, device=self.device)
        M.launch_mesh(verts=pc.verts.detach().reshape(-1, 3), faces=faces, width=self.W, height=self.H,
                      camera=self.cam, adjacency=self._adjacency.get(pc.faces).to(self.device),
                      face_colors=self.face_colors, lighting=self.mesh_lighting, antialias=True, base=base.contiguous(),
                      opacity=self._opacity, out_u8=display, error_flag=self.mesh_error,
                      views=None if self.K == 1 else self.K, quantize=self.quantize)
        return display

    # ---- capture ---------------------------------------------------------------------------------------------------
    def _release(self):
        self.image = self.display = self.radii = self.alpha = self.depth = None
        self.png_out = self.png_len = self._png_scratch = None
        self.mesh_display = self.mesh_png_out = self.mesh_png_len = None

    def _before_capture(self):
        if self.camera is not None:
            self.camera.image_width, self.camera.image_height = self.W, self.H
        if self.mesh:   # the adjacency's build reads sizes on the host: never inside the capture
            self._adjacency.get(self.pc.faces)

    def _after_capture(self):
        # the mesh tensors the replay writes (the model's attributes are replaced by any eager frame)
        self._mesh = tuple(getattr(self.pc, n, None) for n in ("verts", "verts_cano", "face_center", "face_orien_mat",
                                                               "face_scaling")) \
            if self.mesh_update else None
        if self.host_slots:
            self._make_ring()

    def _state_key(self):
        """Beyond the shared key: the image size, `scaling_modifier`, with the mesh overlay what its launch bakes in
        (the faces' address and version, the adjacency, the colour buffer, the lighting) and, with mesh_update=False,
        the addresses of the face frame (and of the vertices the overlay draws) the graph renders."""
        key = super()._state_key() + [self.W, self.H, self.scaling_modifier]
        if self.mesh:
            key += [self.pc.faces.data_ptr(), self.pc.faces._version, self._adjacency.get(self.pc.faces).data_ptr(),
                    None if self.face_colors is None else self.face_colors.data_ptr(), self.mesh_lighting]
            if not self.mesh_update:
                key.append(None if self.pc.verts is None else self.pc.verts.data_ptr())
        if not self.mesh_update and getattr(self.pc, "binding", None) is not None:
            key += [getattr(self.pc, n).data_ptr() for n in ("face_center", "face_orien_mat", "face_scaling")]
        return key

    def _make_ring(self):
        """Pinned host slots, two device staging copies of the display frame and their events."""
        k, shape = self.host_slots, (self.H, self.W, 3) if self.K == 1 else (self.K, self.H, self.W, 3)
        if self.host is None or tuple(self.host[0].shape) != shape:
            torch.cuda.synchronize(self.device)
            self.host = [torch.empty(shape, dtype=torch.uint8).pin_memory() for _ in range(k)]
            self._staged = [torch.empty(shape, dtype=torch.uint8, device=self.device) for _ in range(2)]
        if self.png:   # per slot: K int64 lengths (-1: the replay overflowed), then K files of png_out's stride
            stride = int(self.png_out.shape[1])
            rows = (8 * self.K + stride - 1) // stride + self.K
            if self.host_png_slots is None or tuple(self.host_png_slots[0].shape) != (rows, stride):
                torch.cuda.synchronize(self.device)
                self.host_png_slots = [torch.empty((rows, stride), dtype=torch.uint8).pin_memory() for _ in range(k)]
                self._png_staged = [torch.empty((rows, stride), dtype=torch.uint8, device=self.device)
                                    for _ in range(2)]
            if self.mesh_png_out is not None and (self.host_mesh_png_slots is None or
                                                  tuple(self.host_mesh_png_slots[0].shape) != (rows, stride)):
                # GraphedEval's mesh files travel beside the render's, in the same layout
                torch.cuda.synchronize(self.device)
                self.host_mesh_png_slots = [torch.empty((rows, stride), dtype=torch.uint8).pin_memory()
                                            for _ in range(k)]
                self._mesh_png_staged = [torch.empty((rows, stride), dtype=torch.uint8, device=self.device)
                                         for _ in range(2)]
        self._copy_stream = self._copy_stream or torch.cuda.Stream(device=self.device)
        self._host_events = [None] * k     # per host slot: the copy into it, and which replay it holds
        self._host_replay = [-1] * k
        self._stage_events = [None, None]  # per staging buffer: the copy that last read it

    def _ship(self):
        """Replay i's display frame -> staging buffer i % 2 (on the main stream, right behind the replay) -> host slot
        i % k (copy stream).  The main stream waits only for the copy of replay i - 2, long since done when replays
        take longer than a transfer."""
        i = self.replays - 1
        s, h = i % 2, i % self.host_slots
        cur = torch.cuda.current_stream(self.device)
        if self._stage_events[s] is not None:
            cur.wait_event(self._stage_events[s])
        self._staged[s].copy_(self.display)
        if self.png:   # the compressed bytes only, and -1 for a replay that overflowed (the slot's sticky flag)
            self._png_copy(self.png_out, self.png_len, self._png_staged[s], self.slot.flag)
        if self.mesh_png_out is not None:   # the mesh over the ground truth does not depend on the splats: no flag
            self._png_copy(self.mesh_png_out, self.mesh_png_len, self._mesh_png_staged[s])
        ready = torch.cuda.Event()
        ready.record(cur)
        self._copy_stream.wait_event(ready)
        with torch.cuda.stream(self._copy_stream):
            self.host[h].copy_(self._staged[s], non_blocking=True)
            if self.png:   # staged -> the pinned slot, written by a kernel through its mapped address
                st = self._png_staged[s]
                self._png_copy(self._png_rows(st), self._png_lengths(st), self.host_png_slots[h])
            if self.mesh_png_out is not None:
                st = self._mesh_png_staged[s]
                self._png_copy(self._png_rows(st), self._png_lengths(st), self.host_mesh_png_slots[h])
            done = torch.cuda.Event()
            done.record(self._copy_stream)
        self._stage_events[s] = self._host_events[h] = done
        self._host_replay[h] = i

    def _png_lengths(self, slot):
        """The (K,) int64 lengths at the head of a ring slot."""
        return slot.reshape(-1)[:8 * self.K].view(torch.int64)

    def _png_rows(self, slot):
        """The K file rows at the tail of a ring slot."""
        return slot[slot.shape[0] - self.K:]

    def _png_copy(self, src, src_len, slot, flag=None):
        PNG.launch_copy(src, src_len, self._png_rows(slot), self._png_lengths(slot), flag)

    def host_png(self, replay: Optional[int] = None):
        """Replay `replay`'s PNG file (default: the latest) as bytes -- K files with views_per_replay=K -- once its copy
        has landed.  Raises when that replay overflowed its instance capacity: its frame is incomplete."""
        if not self.png:
            raise ValueError("host_png needs a frame built with png=True")
        return self._host_files(self.host_png_slots, replay, "host_png")

    def _host_files(self, slots, replay, name):
        """Replay `replay`'s files from a ring of PNG slots (one file, or a list of K)."""
        if not self.host_slots:
            raise ValueError(f"{name} needs host_slots > 0")
        i = self.replays - 1 if replay is None else int(replay)
        h = i % self.host_slots
        if self._host_replay[h] != i:
            raise IndexError(f"replay {i} is not in the host ring (slot {h} holds replay {self._host_replay[h]})")
        self._host_events[h].synchronize()
        slot = slots[h]
        lens, rows = self._png_lengths(slot).tolist(), self._png_rows(slot)
        if min(lens) < 0:
            raise RuntimeError(f"{type(self).__name__}: replay {i} overflowed its instance capacity, so its frame is "
                               "incomplete and no PNG file is given for it: regrow() and run it again")
        files = [rows[k, :lens[k]].numpy().tobytes() for k in range(self.K)]
        return files[0] if self.K == 1 else files

    def host_frame(self, replay: Optional[int] = None) -> torch.Tensor:
        """The pinned (H,W,3) uint8 slot ((K,H,W,3) with views_per_replay=K) holding replay `replay` (default: the latest) once its copy has landed."""
        if not self.host_slots:
            raise ValueError("host_frame needs host_slots > 0")
        i = self.replays - 1 if replay is None else int(replay)
        h = i % self.host_slots
        if self._host_replay[h] != i:
            raise IndexError(f"replay {i} is not in the host ring (slot {h} holds replay {self._host_replay[h]})")
        self._host_events[h].synchronize()
        return self.host[h]

    # ---- replay ----------------------------------------------------------------------------------------------------
    def run(self, check: bool = False):
        if self.schedule is not None:   # the schedule's next record
            self._run_scheduled(1, check)
            return self
        if self._stale():
            self.capture()
        self.graph.replay()
        if check and self.overflowed(wait=True):
            self.regrow()
            self.graph.replay()
            if self.overflowed(wait=True):
                raise RuntimeError("GraphedRender: the frame still overflows its instance capacity after re-capture")
        self.replays += 1
        if self.host_slots:
            self._ship()
        return self

    def _replay_scheduled(self):
        self.graph.replay()
        self.replays += 1
        if self.host_slots:
            self._ship()

    def run_iterations(self, n: int, check: bool = True) -> Optional[int]:
        """schedule=: the next n records of the order as n back-to-back replays with no host input (re-capturing first
        if the model changed).  Refused on the host, before anything runs, when they could pass the end of the order.
        check=True synchronises once and regrows after an overflow (see the class documentation).  Returns the number
        of records played (check=True), else None."""
        return self._run_scheduled(n, check)

    def run_all(self, check: bool = True) -> Optional[int]:
        """schedule=: every record of the order not played yet (L replays after set_cursor(0)), as run_iterations."""
        if self.schedule is None:
            raise ValueError("run_all needs a frame built with schedule=")
        return self._run_scheduled(self.schedule.L - self._cursor_host - self._pending, check)


class GraphedEval(GraphedRender):
    """One EVALUATION view as ONE forward-only CUDA graph: a GraphedRender whose captured body ends in the image
    metrics of the rendered view against its ground truth (training.image_metrics, gab200_image_metrics), written into
    row `view` of a (views, 4) device table {l1, psnr, psnr_all, ssim}.  What the reference evaluates per val / test
    view, in training_report (train.py:256-309: select_mesh_by_timestep -> render -> clamp -> l1_loss, psnr, ssim) and
    in render.py + metrics.py (the PNG bytes of every view -> ssim, psnr):

        ev = GraphedEval(pc, width, height, bg, views=len(cams), source="float", warm_cameras=cams)
        for i, cam in enumerate(cams):
            ev.set_inputs(camera=cam, timestep=cam.timestep, gt_u8=gt[i], view=i)   # device buffers: no re-capture
            ev.run()                                                                # enqueue one replay
        s = ev.scores()                    # one synchronisation: s["per_view"], s["l1"], s["psnr"], s["ssim"] ...

    source="float": the graph renders the float image and scores it as train.py does (clamped to [0, 1]; psnr is the
    mean of the three per-channel PSNRs).  source="u8": it renders the display image only (render.py's bytes) and
    scores those as metrics.py reads them back (value/255); `psnr_all` is metrics.py's PSNR (one MSE over all
    values).  With host_slots (source="u8" only) each replay also ships its display frame to the pinned host ring, so
    one replay yields both the PNG bytes render.py would write and the view's scores.  png=True (source="u8") also
    encodes those bytes into a PNG file inside the replay, scores unchanged; host_png(i) returns it.

    camera, timestep, background, ground truth and view index are device buffers written by set_inputs: none of them
    re-captures.  A HOST ground truth (pinned, for an upload that overlaps the replays) travels on a copy stream the
    next replay waits for.  What re-captures is exactly what re-captures a GraphedRender.  The capacity is sized and
    guarded as there; a replay that overflowed its capacity writes no row (the metrics launch reads the slot's sticky
    overflow flag), so a truncated render never produces a score: `scores()` then raises, naming the rows to redo
    after `regrow()`.  `run(check=True)` re-captures and replays an overflowing view at once.

    lpips=net (an lpips.LpipsNet): the body also scores each view's LPIPS distance (gab200_lpips) into row `view` of
    a (views,) device table, with the same rows and the same overflow flag as the metrics; scores() then adds
    `lpips_per_view` and `lpips`.  training_report uses LpipsNet.from_hub_cache("alex"), metrics.py "vgg".

    mesh_opacity=o (source="u8"): render.py's renders_mesh.  After the view is rendered and scored, the body draws the
    mesh of the vertices it posed over the uint8 ground truth `gt` at opacity o (render.py:75-81) into `mesh_display`
    ((H,W,3), or (K,H,W,3) in one K-view call); scores and `display` are those of the frame without it.  With png=True
    it is also encoded into `mesh_png_out` / `mesh_png_len`, and with host_slots those files travel in the ring beside
    the render's: host_mesh_png(i).  The mesh frame does not depend on the splats, so a replay that overflowed its
    capacity still draws (and ships) it.  face_colors and mesh_lighting mean what they mean for a GraphedRender."""

    _MESH_OVER_GT = True

    def __init__(self, pc, width: int, height: int, bg: torch.Tensor, views: int, source: str = "float",
                 host_slots: int = 0, capacity: Optional[int] = None, headroom: float = 1.25, warm_cameras=None,
                 warm_timesteps=None, views_per_replay: int = 1, schedule=None, frames=None, lpips=None,
                 png: bool = False, mesh_opacity: Optional[float] = None, face_colors: Optional[torch.Tensor] = None,
                 mesh_lighting: str = "front"):
        """views_per_replay=K > 1: one replay renders K cameras of one timestep in one forward and scores them into
        rows view .. view + K - 1 (set_inputs(cameras=K cameras, gt_u8=(K,3,H,W), view=first row)); warm_cameras is a
        list of K-camera groups.  K is fixed per capture: a last group of fewer views is the business of a
        single-view (or smaller) GraphedEval.
        schedule=s with frames=store (a schedule.ViewSchedule of R records of K cameras, and the FrameStore its ids
        index; views >= R * K): every replay runs the next record of the schedule with no host input.  A sampler kernel
        copies record r = order[cursor] into the camera table, the timestep, the frame ids and the rows r * K ..
        r * K + K - 1; the store's decode writes `gt`; the view is rendered and scored into those rows; a commit kernel
        advances the cursor unless the replay overflowed.  run_all() scores the rest of the order; reset() also
        rewinds the cursor; set_inputs is refused.  The warm-up renders `warm_cameras` if given, else up to 16 records
        at their own timesteps."""
        if source not in ("float", "u8"):
            raise ValueError("source must be 'float' (train.py's evaluation of the float render) or 'u8' (the "
                             "display bytes render.py writes, scored as metrics.py reads them)")
        if host_slots and source != "u8":
            raise ValueError("host_slots ships the display image: it needs source='u8'")
        if png and source != "u8":
            raise ValueError("png=True encodes the display image: it needs source='u8'")
        if mesh_opacity is not None and source != "u8":
            raise ValueError("mesh_opacity draws render.py's renders_mesh over the uint8 ground truth: it needs "
                             "source='u8'")
        if int(views) < 1:
            raise ValueError("views must be at least 1")
        if isinstance(views_per_replay, int) and views_per_replay > int(views):
            raise ValueError(f"views_per_replay={views_per_replay} exceeds the table's {int(views)} rows")
        if lpips is not None:
            if not isinstance(lpips, LpipsNet):
                raise TypeError(f"lpips must be an LpipsNet, got {type(lpips).__name__}")
            if min(int(width), int(height)) < lpips.min_side:
                raise ValueError(f"LPIPS with {lpips.net} needs an image of at least {lpips.min_side}x"
                                 f"{lpips.min_side} pixels, got {int(width)}x{int(height)}")
        super().__init__(pc, width, height, bg, outputs="float" if source == "float" else "u8", host_slots=host_slots,
                         capacity=capacity, headroom=headroom, warm_cameras=warm_cameras, warm_timesteps=warm_timesteps,
                         views_per_replay=views_per_replay, png=png, mesh_opacity=mesh_opacity,
                         face_colors=face_colors, mesh_lighting=mesh_lighting)
        self.source, self.views = source, int(views)
        self.table = torch.empty((self.views, N.METRICS_FIELDS), dtype=torch.float32, device=self.device)
        if lpips is not None and lpips.device != self.device:
            raise ValueError(f"the LpipsNet is on {lpips.device}, the model on {self.device}")
        self.lpips = lpips
        self.lpips_table = torch.empty(self.views, dtype=torch.float32, device=self.device) \
            if lpips is not None else None
        self.frames = frames
        self.frame_ids = None
        if (schedule is None) != (frames is None):
            raise ValueError("a GraphedEval scores a schedule's records against their frames: give schedule= and "
                             "frames= together")
        if schedule is not None:
            self._check_store(frames)
            self._use_schedule(schedule, frames, log=False)
            if schedule.R * self.K > self.views:
                raise ValueError(f"the schedule's {schedule.R} records of {self.K} views score {schedule.R * self.K} "
                                 f"rows, the table has {self.views}")
            self.frame_ids = torch.zeros(self.K, dtype=torch.int32, device=self.device)
        self.reset()
        self.view = torch.zeros(1, dtype=torch.int32, device=self.device)
        # K > 1: the rows of the replay's views, view + k, one device int32 each
        self.rows = torch.arange(self.K, dtype=torch.int32, device=self.device) if self.K > 1 else None
        self.gt = torch.zeros(self._gt_shape(), dtype=torch.uint8, device=self.device)

    def reset(self):
        """Every row of the tables back to NaN (no score); with a schedule, the cursor back to its first record."""
        self.table.fill_(float("nan"))
        if self.lpips_table is not None:
            self.lpips_table.fill_(float("nan"))
        if self.schedule is not None:
            self.set_cursor(0)

    # ---- inputs ------------------------------------------------------------------------------------------------
    def set_inputs(self, camera=None, timestep=None, gt_u8=None, view=None, verts=None, bg=None, cameras=None,
                   mesh_opacity=None, face_colors=None):
        """As GraphedRender.set_inputs, plus the view's ground truth (uint8 (3,H,W), a device tensor or a pinned host
        tensor) and its row in the table (a host int in [0, views)).  None of them re-captures.  views_per_replay=K >
        1: `cameras` (K), gt_u8 (K,3,H,W), and `view` is the first of the K rows (view + K <= views)."""
        if self.schedule is not None:
            raise ValueError("this GraphedEval samples every input from its schedule on the device: set_inputs is "
                             "refused (reset() or set_cursor() move it)")
        if view is not None:
            view = int(view)
            if not 0 <= view <= self.views - self.K:
                raise IndexError(f"rows {view} .. {view + self.K - 1} outside the table's {self.views} rows")
        group = camera if self.K == 1 else (None if cameras is None or isinstance(cameras, torch.Tensor)
                                            else list(cameras)[0])
        size = (int(group.image_height), int(group.image_width)) \
            if group is not None and not isinstance(group, torch.Tensor) else (self.H, self.W)
        want = (3, *size) if self.K == 1 else (self.K, 3, *size)
        if gt_u8 is not None and (gt_u8.dtype != torch.uint8 or tuple(gt_u8.shape) != want):
            raise ValueError(f"gt_u8 must be a uint8 {want} tensor, got {gt_u8.dtype} {tuple(gt_u8.shape)}")
        super().set_inputs(camera=camera, timestep=timestep, verts=verts, bg=bg, cameras=cameras,
                           mesh_opacity=mesh_opacity, face_colors=face_colors)
        if tuple(self.gt.shape) != self._gt_shape():   # a camera of another size (the next run() re-captures)
            self._await_upload()
            self.gt = torch.zeros(self._gt_shape(), dtype=torch.uint8, device=self.device)
        if gt_u8 is not None:
            if gt_u8.device.type == "cpu" and self.device.type == "cuda":
                if self._side is None:
                    self._side = torch.cuda.Stream(device=self.device)
                self._upload(self.gt, gt_u8)
            else:
                self._await_upload()   # an earlier host upload must not land after this copy
                self.gt.copy_(gt_u8, non_blocking=True)
        if view is not None:
            self.view.fill_(view)
            if self.rows is not None:
                self.rows.copy_(torch.arange(view, view + self.K, dtype=torch.int32), non_blocking=True)

    # ---- the frame body: the playback frame, then the metrics of what it rendered ------------------------------
    def _body(self, captured: bool = False):
        if captured and self.schedule is not None:   # this replay's record, its rows, and its ground truth
            self._launch_sample(ids=self.frame_ids, rows=self.view if self.K == 1 else self.rows)
            self.frames.launch_decode(self.frame_ids, self.gt, None)
        self._frame(captured)
        if captured:   # the warm-up frames score nothing: they would write the current view's row
            rendered = self.image if self.source == "float" else self.display
            if self.K == 1:
                launch_image_metrics(rendered, self.gt, self.table, row=self.view, skip_flag=self.slot.flag,
                                     scratch=self._metrics_scratch)
            else:   # one launch per view, each into its own row; an overflowed replay writes none of them
                for k in range(self.K):
                    launch_image_metrics(rendered[k], self.gt[k], self.table, row=self.rows[k:k + 1],
                                         skip_flag=self.slot.flag, scratch=self._metrics_scratch)
            if self.lpips is not None:   # after the metrics, into the same rows, under the same flag
                for k in range(self.K):
                    launch_lpips(rendered if self.K == 1 else rendered[k], self.gt if self.K == 1 else self.gt[k],
                                 self.lpips, self.lpips_table, row=self.view if self.K == 1 else self.rows[k:k + 1],
                                 skip_flag=self.slot.flag, scratch=self._lpips_scratch)
            if self.mesh:   # render.py's renders_mesh: over the ground truth, whatever the splats did
                with torch.no_grad():
                    self.mesh_display = self._overlay(self.gt)
                if self.png:
                    self.mesh_png_out, self.mesh_png_len = self._encode(self.mesh_display)
            if self.schedule is not None:
                self._launch_commit()

    def _before_capture(self):
        super()._before_capture()
        self._metrics_scratch = metrics_scratch(self.H, self.W, self.device)
        self._lpips_scratch = lpips_scratch(self.lpips, self.H, self.W) if self.lpips is not None else None

    def _state_key(self):
        """Beyond a GraphedRender's key: with a frame store, the addresses of its arena and index; with LPIPS, the
        address of the packed weights."""
        key = super()._state_key()
        if self.frames is not None:
            key.append(self.frames.pointers())
        if self.lpips is not None:
            key.append(self.lpips.weights.data_ptr())
        return key

    # ---- replay ----------------------------------------------------------------------------------------------------
    def run(self, check: bool = False):
        if self.schedule is not None:   # the schedule's next record
            self._run_scheduled(1, check)
            return self
        self._await_upload()
        super().run(check)
        if self._side is not None:
            self._mark_read()
        return self

    def host_mesh_png(self, replay: Optional[int] = None):
        """Replay `replay`'s mesh PNG file (default: the latest) as bytes -- K files with views_per_replay=K -- once its
        copy has landed: render.py's renders_mesh/*.png.  Given for an overflowed replay too (the mesh frame does not
        depend on the splats)."""
        if not (self.mesh and self.png):
            raise ValueError("host_mesh_png needs a GraphedEval built with mesh_opacity= and png=True")
        return self._host_files(self.host_mesh_png_slots, replay, "host_mesh_png")

    def run_all(self, check: bool = True) -> Optional[int]:
        """schedule=: scores every record of the order not scored yet, as back-to-back replays with no host input (R
        replays after reset() with the identity order).  check=True synchronises once; a replay that overflowed its
        capacity wrote no row and committed nothing, nor did the replays behind it, so the frame regrows and redoes
        the records from the cursor on.  Returns the number of records scored (check=True), else None."""
        if self.schedule is None:
            raise ValueError("run_all needs a GraphedEval built with schedule= and frames=")
        return self._run_scheduled(self.schedule.L - self._cursor_host - self._pending, check)

    def scores(self, n: Optional[int] = None) -> dict:
        """Synchronises once and returns the first n rows (default: all): `per_view`, a (n, 4) float32 host tensor
        {l1, psnr, psnr_all, ssim}, and the mean of each column as training_report forms its means (the per-view floats
        summed in double, then divided by n: train.py:286-303).  `psnr` is train.py's PSNR, `psnr_all` metrics.py's.
        With lpips=: `lpips_per_view`, a (n,) float32 host tensor, and `lpips`, its mean formed the same way.
        Raises if a requested row holds no score (NaN): its replay overflowed the capacity (run(check=False)), or the
        view was never run."""
        n = self.views if n is None else int(n)
        if not 1 <= n <= self.views:
            raise IndexError(f"n must lie in [1, {self.views}]")
        rows = self.table[:n].cpu()
        nan = torch.isnan(rows).any(dim=1)
        if self.lpips_table is not None:
            lp = self.lpips_table[:n].cpu()
            nan |= torch.isnan(lp)
        missing = nan.nonzero().flatten().tolist()
        if missing:
            raise RuntimeError(f"GraphedEval: rows {missing} hold no score -- their replay overflowed the instance "
                               "capacity (run(check=False)) or never ran: call regrow() and run those views again")
        out = {"per_view": rows}
        for i, name in enumerate(METRIC_NAMES):
            total = 0.0
            for v in rows[:, i].tolist():
                total += v
            out[name] = total / n
        if self.lpips_table is not None:
            out["lpips_per_view"] = lp
            total = 0.0
            for v in lp.tolist():
                total += v
            out["lpips"] = total / n
        return out
