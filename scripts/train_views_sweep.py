"""Per-view cost of a training iteration over the cameras of one timestep K at a time (GraphedFrame(views_per_replay=K),
one forward + backward for the K views, one optimiser step) against one iteration per camera -> one JSON line per
(setting, K, arm) on stdout (profiles/h100/train_views.jsonl):

  graph_full_flame_single   GraphedFrame: one replay per view (FLAME pose + face frame + render + photometric loss +
                            regularisers + backward + densification statistics + capturable Adam over the splat and
                            FLAME groups)
  graph_full_flame_views    the same iteration with views_per_replay=K: one replay per K views of a timestep

A pass is 16 cameras (distinct fields of view) x 2 FLAME timesteps = 32 views; the arms run alternately in one process,
3 passes each after a warm-up pass, and each line reports the median per-view time.  Settings: the demo size (550x802,
89,021 splats) and 150k splats at 1920x1080, K in {1, 4, 16}.  Then one torch.profiler line per setting: the kernel time
per view of one pass of each arm at K = 16, so the saving can be attributed (FLAME pose, Adam, preprocess backward,
...).  Every line carries the card, its power limit and its SM clock, read in the same run."""
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import gaussianavatars_b200 as g  # noqa: E402
from gaussianavatars_b200 import synthetic as syn  # noqa: E402
from gaussianavatars_b200.flame import FlameLBS  # noqa: E402
from gaussianavatars_b200.graph import GraphedFrame  # noqa: E402
from gaussianavatars_b200.model import MeshBoundGaussians  # noqa: E402

dev = torch.device("cuda:0")
STEPS = (0, 5)
VIEWS = 16 * len(STEPS)
LRS = {"xyz": 1.6e-4, "rotation": 1e-3, "scaling": 5e-3, "opacity": 5e-2, "f_dc": 2.5e-3, "f_rest": 1.25e-4}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    if len(q) == 3:
        return {"gpu": q[0], "power_limit_W": float(q[1]), "sm_clock_MHz": float(q[2])}
    return {"gpu": torch.cuda.get_device_name(dev)}


def rig(W, H, n=16):
    cams = []
    for i in range(n):
        orb = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=-50 + 100 * i / (n - 1),
                               elevation_deg=6 * math.sin(i))
        f = 1.0 + 0.08 * (2 * i / (n - 1) - 1)
        cams.append(syn.look_at_camera(W, H, math.degrees(orb.FoVx) * f, math.degrees(orb.FoVy) * f,
                                       w2c=orb.world_view_transform.T.numpy()).to(dev))
    return cams


def setting(P, W, H, T=8):
    a = syn.flame_like_assets(0)
    fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0]).items()
          if k != "dynamic_offset"}
    lbs = FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                               a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, None, None, device=dev, requires_grad=True, flame=lbs, flame_param=fp)
    for attr in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest"):
        setattr(pc, attr, torch.nn.Parameter(getattr(pc, attr).detach().clone()))
    groups = [{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pc.parameters())]
    opt = g.Adam(groups + g.flame_param_groups(pc.flame_param), lr=0.0, eps=1e-15, capturable=True)
    for n in ("xyz_gradient_accum", "denom"):
        setattr(pc, n, torch.zeros((P, 1), device=dev))
    pc.max_radii2D = torch.zeros((P,), device=dev)
    gts = torch.randint(0, 256, (16, 3, H, W), generator=torch.Generator().manual_seed(11), dtype=torch.uint8).to(dev)
    return pc, opt, rig(W, H), gts


def frame(pc, opt, W, H, K, warm):
    return GraphedFrame(pc, W, H, 1.0, 1.0, torch.ones(3), loss="photometric", regularizers={}, optimizer=opt,
                        densify_stats=True, per_camera_fov=True, views_per_replay=K, warm_cameras=warm)


def arms(pc, opt, cams, gts, W, H, K):
    single = frame(pc, opt, W, H, 1, cams)
    groups = [cams[i:i + K] for i in range(0, 16, K)]
    views = frame(pc, opt, W, H, K, groups if K > 1 else cams)   # K = 1: the single-view frame, a second instance

    def run_single():
        for t in STEPS:
            for i, c in enumerate(cams):
                single.set_inputs(camera=c, timestep=t, gt_u8=gts[i])
                single.run()

    def run_views():
        for t in STEPS:
            for j, grp in enumerate(groups):
                if K > 1:
                    views.set_inputs(cameras=grp, timestep=t, gt_u8=gts[j * K:(j + 1) * K])
                else:
                    views.set_inputs(camera=grp[0], timestep=t, gt_u8=gts[j])
                views.run()
    return {"graph_full_flame_single": run_single, "graph_full_flame_views": run_views}, [single, views]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def sweep(name, P, W, H, info):
    pc, opt, cams, gts = setting(P, W, H)
    for K in (1, 4, 16):
        fns, frames = arms(pc, opt, cams, gts, W, H, K)
        for fn in fns.values():   # warm-up pass (captures)
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in fns}
        for _ in range(3):   # the arms alternate, pass by pass
            for k, fn in fns.items():
                ms[k].append(timed(fn))
        overflow = any(f.overflowed() for f in frames)
        for arm, v in ms.items():
            v = sorted(v)
            print(json.dumps({"setting": name, "splats": P, "W": W, "H": H, "K": K, "arm": arm,
                              "views_per_pass": VIEWS, "ms_per_view_median": round(v[1] / VIEWS, 4),
                              "ms_per_view_best": round(v[0] / VIEWS, 4), "passes": 3, "overflow": overflow,
                              "captures": [f.captures for f in frames], **info}), flush=True)
        if K == 16:
            profile(name, P, W, H, fns, info)
        del fns, frames
        torch.cuda.empty_cache()


def profile(name, P, W, H, fns, info):
    from torch.profiler import ProfilerActivity, profile as prof_ctx
    line = {"setting": name, "splats": P, "W": W, "H": H, "K": 16, "arm": "profile", "views_per_pass": VIEWS}
    for arm, fn in fns.items():
        with prof_ctx(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                short = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("gab::", "")[:60]
                kern[short] = kern.get(short, 0.0) + e.device_time_total
        top = sorted(kern.items(), key=lambda kv: -kv[1])
        line[arm + "_kernel_us_per_view"] = {k: round(v / VIEWS, 2) for k, v in top[:16]}
        line[arm + "_total_kernel_us_per_view"] = round(sum(kern.values()) / VIEWS, 2)
    print(json.dumps({**line, **info}), flush=True)


def main():
    info = gpu_info()
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p_150k", 150_000, 1920, 1080)):
        sweep(name, P, W, H, info)


if __name__ == "__main__":
    main()
