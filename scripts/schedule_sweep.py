"""What sampling the iteration's inputs on the device costs and saves -> one JSON line per measurement on stdout
(profiles/h100/schedule.jsonl):

  iteration   time per iteration of the captured FLAME training iteration with frames=store (GraphedFrame: pose +
              decode + render + photometric loss + regularisers + backward + densification statistics + capturable
              Adam), two arms over the same iterations:
                (b) store      set_inputs(camera table already on the device, timestep, K ids) then run(), per iteration
                (c) schedule   a ViewSchedule of the same iterations: set_cursor(0), then run_iterations(n,
                               check=False) -- n back-to-back replays, no host input
              A pass is 16 cameras x 2 FLAME timesteps = 32 views, K views per replay; the arms alternate pass by pass,
              5 passes each after a warm-up pass; median, min and max.  `host_ms_per_iter` is the host time spent
              enqueueing one iteration, median over the passes.
  kernels     gab200_schedule_sample and gab200_schedule_commit alone: CUDA events around 1000 launches each, per
              launch, median of 5.

Settings: the demo (550x802, 89,021 splats) and 100k splats at 1920x1080, K in {1, 16}.  Every line carries the card,
its power limit and its SM clock, read in the same run."""
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import gaussianavatars_b200 as g  # noqa: E402
from gaussianavatars_b200 import _native as N  # noqa: E402
from gaussianavatars_b200.graph import GraphedFrame, camera_block  # noqa: E402
from scripts.rgba_mask_sweep import rgba_frames  # noqa: E402
from scripts.train_views_sweep import gpu_info, setting, timed  # noqa: E402

dev = torch.device("cuda:0")
STEPS = (0, 5)
VIEWS = 16 * len(STEPS)
PASSES = 5


def iteration_arms(pc, opt, cams, store, W, H, K):
    groups = [cams[i:i + K] for i in range(0, 16, K)]
    warm = groups if K > 1 else cams
    kw = dict(loss="photometric", regularizers={}, optimizer=opt, densify_stats=True, per_camera_fov=True,
              views_per_replay=K, warm_cameras=warm, frames=store)
    work = [(t, j) for t in STEPS for j in range(len(groups))]
    st = GraphedFrame(pc, W, H, 1.0, 1.0, torch.ones(3), **kw)
    sched = g.ViewSchedule([groups[j] if K > 1 else groups[j][0] for _, j in work], timesteps=[t for t, _ in work],
                           frames=[list(range(j * K, (j + 1) * K)) if K > 1 else j for _, j in work], device=dev)
    sc = GraphedFrame(pc, W, H, 1.0, 1.0, torch.ones(3), schedule=sched, **kw)
    tables = [torch.stack([camera_block(c, fov=True) for c in grp]).reshape(st.cam.shape).to(dev) for grp in groups]
    host = {"store": [], "schedule": []}

    def run_store():
        t0 = time.perf_counter()
        for t, j in work:
            ids = list(range(j * K, (j + 1) * K))
            if K > 1:
                st.set_inputs(cameras=tables[j], timestep=t, frames=ids)
            else:
                st.set_inputs(camera=tables[j], timestep=t, frames=ids[0])
            st.run()
        host["store"].append((time.perf_counter() - t0) * 1e3 / len(work))

    def run_schedule():
        t0 = time.perf_counter()
        sc.set_cursor(0)
        sc.run_iterations(len(work), check=False)
        host["schedule"].append((time.perf_counter() - t0) * 1e3 / len(work))
    return {"store": run_store, "schedule": run_schedule}, [st, sc], host


def kernel_lines(info):
    """The two kernels alone, at K = 1 and 16, from a table of 64 records."""
    out = []
    L_ = N.lib()
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for K in (1, 16):
        R = 64
        cams = torch.randn(R, K, 37, device=dev)
        ts = torch.zeros(R, dtype=torch.int32, device=dev)
        fids = torch.zeros(R, K, dtype=torch.int32, device=dev)
        order = torch.arange(R, dtype=torch.int32, device=dev)
        cursor = torch.zeros(1, dtype=torch.int32, device=dev)
        cam_out = torch.empty(K, 37, device=dev)
        t_out, exhausted, flag = (torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(3))
        ids_out = torch.empty(K, dtype=torch.int32, device=dev)
        loss = torch.zeros((), device=dev)
        losses = torch.zeros(R, device=dev)
        n = 1000

        def samples():
            for _ in range(n):
                L_.gab200_schedule_sample(R, K, R, cams.data_ptr(), ts.data_ptr(), fids.data_ptr(), order.data_ptr(),
                                          cursor.data_ptr(), cam_out.data_ptr(), t_out.data_ptr(), ids_out.data_ptr(),
                                          None, exhausted.data_ptr(), stream)

        def commits():   # the overflow flag set: the commit reads it and writes nothing, so the cursor stays in range
            for _ in range(n):
                L_.gab200_schedule_commit(R, flag.data_ptr(), exhausted.data_ptr(), loss.data_ptr(),
                                          losses.data_ptr(), cursor.data_ptr(), stream)
        flag.fill_(1)
        for name, fn in (("sample", samples), ("commit", commits)):
            fn()
            ms = sorted(timed(fn) for _ in range(5))
            out.append(dict(arm="kernel", kernel=f"gab200_schedule_{name}", K=K, launches=n,
                            us_per_launch_median=round(ms[2] * 1e3 / n, 3), us_per_launch_min=round(ms[0] * 1e3 / n, 3),
                            us_per_launch_max=round(ms[-1] * 1e3 / n, 3), **info))
    return out


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    for rec in kernel_lines(info):
        emit(rec)
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p", 100_000, 1920, 1080)):
        pc, opt, cams, _ = setting(P, W, H)
        store = g.FrameStore(W, H, [1.0, 1.0, 1.0], dev)
        store.add_rgba(rgba_frames(16, H, W).to(dev))
        for K in (1, 16):
            fns, frames, host = iteration_arms(pc, opt, cams, store, W, H, K)
            for fn in fns.values():   # warm-up pass (captures)
                fn()
            torch.cuda.synchronize()
            for v in host.values():
                v.clear()
            ms = {k: [] for k in fns}
            for _ in range(PASSES):
                for k, fn in fns.items():
                    ms[k].append(timed(fn))
            overflow = any(f.overflowed() for f in frames)
            iters = VIEWS // K
            for arm, v in ms.items():
                v, hv = sorted(v), sorted(host[arm])
                emit({"setting": name, "splats": P, "W": W, "H": H, "K": K, "arm": arm, "iterations_per_pass": iters,
                      "ms_per_iter_median": round(v[len(v) // 2] / iters, 4), "ms_per_iter_min": round(v[0] / iters, 4),
                      "ms_per_iter_max": round(v[-1] / iters, 4), "host_ms_per_iter_median": round(hv[len(hv) // 2], 4),
                      "passes": len(v), "overflow": overflow, "captures": [f.captures for f in frames], **info})
            del fns, frames
            torch.cuda.empty_cache()
        del pc, opt, store
        torch.cuda.empty_cache()
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
