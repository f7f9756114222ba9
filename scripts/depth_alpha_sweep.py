"""Cost of the alpha and depth planes -> one JSON line per (setting, arm, depth_alpha) on stdout
(profiles/h100/depth_alpha.jsonl):

  replay_u8   GraphedRender(outputs="u8"[, depth_alpha=True]): one playback replay per view
  step        eager render(..., depth_alpha) + an L1 loss [+ a term on alpha and depth] + backward, per view

A pass is 16 cameras x 4 FLAME timesteps (replays) or 16 cameras at one timestep (steps); the two forms of each arm
run alternately in one process, 5 passes each after a warm-up pass, and each line reports the median per-view time
and the spread of the passes.  Settings: the demo (550x802, 89,021 splats) and 100k splats at 1920x1080.  Every line
carries the card, its power limit and its SM clock, read in the same run."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

from scripts.multiview_sweep import gpu_info, setting, timed  # noqa: E402
from gaussianavatars_b200.graph import GraphedRender  # noqa: E402
from gaussianavatars_b200.renderer import render  # noqa: E402

dev = torch.device("cuda:0")
STEPS = (0, 5, 10, 15)


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def arms(pc, cams, gts, W, H):
    bg = torch.ones(3, device=dev)
    out = {}
    for da in (False, True):
        g = GraphedRender(pc, W, H, bg, outputs="u8", warm_cameras=cams, warm_timesteps=STEPS, depth_alpha=da)

        def replay(g=g):
            for t in STEPS:
                for c in cams:
                    g.set_inputs(camera=c, timestep=t)
                    g.run()
        out[("replay_u8", da)] = (replay, len(STEPS) * len(cams), g)

    gts_f = gts.float() / 255.0
    mask = (gts_f.mean(1, keepdim=True) > 0.5).float()

    def step(da):
        def run():
            pc.select_mesh_by_timestep(0)
            for i, c in enumerate(cams):
                o = render(c, pc, Pipe, bg, depth_alpha=da)
                loss = (o["render"] - gts_f[i]).abs().mean()
                if da:
                    loss = loss + 0.1 * (o["alpha"] - mask[i]).abs().mean() + 1e-3 * o["depth"].mean()
                loss.backward()
        return run
    out[("step", False)] = (step(False), len(cams), None)
    out[("step", True)] = (step(True), len(cams), None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the lines to this file")
    args = ap.parse_args()
    info = gpu_info()
    lines = []
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p", 100_000, 1920, 1080)):
        pc, cams, gts = setting(P, W, H)
        a = arms(pc, cams, gts, W, H)
        for fn, _, _ in a.values():   # warm-up pass (captures, allocator, autotuning)
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in a}
        for _ in range(args.passes):   # the arms alternate pass by pass
            for k, (fn, _, _) in a.items():
                ms[k] += timed(fn, passes=1)
        for (arm, da), (fn, views, g) in a.items():
            t = sorted(ms[(arm, da)])
            rec = dict(setting=name, P=P, W=W, H=H, arm=arm, depth_alpha=da, views_per_pass=views,
                       ms_per_view_median=t[len(t) // 2] / views, ms_per_view_min=t[0] / views,
                       ms_per_view_max=t[-1] / views, passes=len(t), **info)
            if g is not None:
                rec["captures"] = g.captures
                rec["overflowed"] = bool(g.overflowed())
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        del a, pc
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
