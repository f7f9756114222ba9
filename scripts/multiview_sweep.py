"""Per-view cost of rendering (and scoring) the cameras of one timestep K at a time in one replay, against one replay per
camera -> one JSON line per (setting, K, arm) on stdout (profiles/h100/multiview.jsonl):

  render_single   GraphedRender, outputs "u8": one replay per view (set_inputs(camera, timestep), run)
  render_views    GraphedRender(views_per_replay=K): one replay per K views of a timestep
  eval_single     GraphedEval (source "float"): one replay per view, metrics into the view's row
  eval_views      GraphedEval(views_per_replay=K): one replay scores K views

A pass is 16 cameras (distinct fields of view) x 4 FLAME timesteps = 64 views; the arms run alternately in one
process, 3 passes each after a warm-up pass, and each line reports the median per-view time.  Settings: the demo
(550x802, 89,021 splats, a FLAME head with 16 timesteps) and 100k splats at 1920x1080.  With --profile the script
instead records torch.profiler kernel times of one pass of 16-view render replays per setting.  Every line carries the
card, its power limit and its SM clock, read in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

from gaussianavatars_b200 import synthetic as syn  # noqa: E402
from gaussianavatars_b200.flame import FlameLBS  # noqa: E402
from gaussianavatars_b200.graph import GraphedEval, GraphedRender  # noqa: E402
from gaussianavatars_b200.model import MeshBoundGaussians  # noqa: E402

dev = torch.device("cuda:0")
STEPS = (0, 5, 10, 15)


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


def setting(P, W, H, T=16):
    a = syn.flame_like_assets(0)
    fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0]).items()
          if k != "dynamic_offset"}
    lbs = FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                               a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, None, None, device=dev, flame=lbs, flame_param=fp)
    g = torch.Generator().manual_seed(11)
    gts = torch.randint(0, 256, (16, 3, H, W), generator=g, dtype=torch.uint8).to(dev)
    return pc, rig(W, H), gts


def timed(fn, passes=3):
    ms = []
    for _ in range(passes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return sorted(ms)


def arms(pc, cams, gts, W, H, K):
    bg = torch.ones(3, device=dev)
    groups = [cams[i:i + K] for i in range(0, 16, K)]
    out = {}
    rs = GraphedRender(pc, W, H, bg, outputs="u8", warm_cameras=cams, warm_timesteps=STEPS)
    es = GraphedEval(pc, W, H, bg, views=16, warm_cameras=cams, warm_timesteps=STEPS)

    def render_single():
        for t in STEPS:
            for c in cams:
                rs.set_inputs(camera=c, timestep=t)
                rs.run()

    def eval_single():
        for t in STEPS:
            for i, c in enumerate(cams):
                es.set_inputs(camera=c, timestep=t, gt_u8=gts[i], view=i)
                es.run()
    out["render_single"], out["eval_single"] = render_single, eval_single
    graphs = [rs, es]
    if K > 1:
        rv = GraphedRender(pc, W, H, bg, outputs="u8", views_per_replay=K, warm_cameras=groups, warm_timesteps=STEPS)
        ev = GraphedEval(pc, W, H, bg, views=16, views_per_replay=K, warm_cameras=groups, warm_timesteps=STEPS)

        def render_views():
            for t in STEPS:
                for grp in groups:
                    rv.set_inputs(cameras=grp, timestep=t)
                    rv.run()

        def eval_views():
            for t in STEPS:
                for j, grp in enumerate(groups):
                    ev.set_inputs(cameras=grp, timestep=t, gt_u8=gts[j * K:(j + 1) * K], view=j * K)
                    ev.run()
        out["render_views"], out["eval_views"] = render_views, eval_views
        graphs += [rv, ev]
    return out, graphs


def sweep(settings, info):
    for name, P, W, H in settings:
        pc, cams, gts = setting(P, W, H)
        for K in (1, 4, 16):
            fns, graphs = arms(pc, cams, gts, W, H, K)
            for fn in fns.values():   # warm-up pass (captures)
                fn()
            torch.cuda.synchronize()
            ms = {k: [] for k in fns}
            for _ in range(3):   # the arms alternate, pass by pass
                for k, fn in fns.items():
                    ms[k] += timed(fn, passes=1)
            assert not any(g.overflowed() for g in graphs) and all(g.captures == 1 for g in graphs)
            for arm, v in ms.items():
                v = sorted(v)
                print(json.dumps({"setting": name, "splats": P, "W": W, "H": H, "K": K, "arm": arm,
                                  "views_per_pass": 64, "ms_per_view_median": round(v[1] / 64, 4),
                                  "ms_per_view_best": round(v[0] / 64, 4), "passes": 3, **info}), flush=True)
            del fns, graphs
            torch.cuda.empty_cache()


def profile(settings, info):
    from torch.profiler import ProfilerActivity, profile as prof_ctx
    for name, P, W, H in settings:
        pc, cams, gts = setting(P, W, H)
        fns, graphs = arms(pc, cams, gts, W, H, 16)
        for arm in ("render_single", "render_views"):
            fns[arm]()
            torch.cuda.synchronize()
            with prof_ctx(activities=[ProfilerActivity.CUDA]) as prof:
                fns[arm]()
                torch.cuda.synchronize()
            kern = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    short = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("gab::", "")[:60]
                    k = kern.setdefault(short, [0.0, 0])
                    k[0] += e.device_time_total
                    k[1] += e.count
            replays = 64 if arm == "render_single" else 4
            top = sorted(kern.items(), key=lambda kv: -kv[1][0])
            print(json.dumps({"setting": name, "splats": P, "W": W, "H": H, "K": 16, "arm": "profile_" + arm,
                              "replays": replays,
                              "kernel_us_per_replay": {k: round(v[0] / replays, 2) for k, v in top[:14]},
                              "tile_scan_order_us_per_launch": round(kern.get("tile_scan_order_kernel", [0, 1])[0] /
                                                                     max(kern.get("tile_scan_order_kernel", [0, 1])[1], 1), 2),
                              **info}), flush=True)
        del fns, graphs
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    settings = (("demo", 89_021, 550, 802), ("1080p_100k", 100_000, 1920, 1080))
    info = gpu_info()
    (profile if args.profile else sweep)(settings, info)


if __name__ == "__main__":
    main()
