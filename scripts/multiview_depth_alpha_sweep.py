"""Cost of the alpha and depth planes on K-view frames -> one JSON line per (setting, K, arm) on stdout
(profiles/h100/multiview_depth_alpha.jsonl):

  forward
    single_display_da   K x render_display(depth_alpha=True)
    views_da            one render_views(depth_alpha=True) of the K cameras
    views               one render_views of the K cameras, no planes
  training step (eager, one FLAME timestep; loss = L1 [+ 0.1 x L1(alpha, mask) + 1e-3 x mean(depth)], then backward)
    single_step_da      K x render(depth_alpha=True) + the loss + backward
    views_step_da       one render_views_train(depth_alpha=True) + the same loss over the K views + backward
    views_step          one render_views_train + the L1 loss + backward, no planes

A pass renders the 16 cameras of the rig in 16 / K groups of K; the arms alternate pass by pass in one process,
`--passes` passes each after a warm-up pass, and each line reports the median per-view time and the spread of the
passes.  Settings: the demo (550x802, 89,021 splats) and 100k splats at 1920x1080; K = 4 and 16.  Every line carries
the card, its power limit and its SM clock, read in the same run."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

from scripts.multiview_sweep import gpu_info, setting, timed  # noqa: E402
from gaussianavatars_b200.renderer import render, render_display, render_views, render_views_train  # noqa: E402

dev = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def arms(pc, cams, gts, K):
    bg = torch.ones(3, device=dev)
    groups = [cams[i:i + K] for i in range(0, len(cams), K)]
    gts_f = gts.float() / 255.0
    mask = (gts_f.mean(1, keepdim=True) > 0.5).float()

    def loss_of(img, gt, m, alpha=None, depth=None):
        loss = (img - gt).abs().mean()
        if alpha is not None:
            loss = loss + 0.1 * (alpha - m).abs().mean() + 1e-3 * depth.mean()
        return loss

    def single_display_da():
        with torch.no_grad():
            for c in cams:
                render_display(c, pc, Pipe, bg, depth_alpha=True)

    def views_forward(da):
        def run():
            with torch.no_grad():
                for g in groups:
                    render_views(g, pc, Pipe, bg, depth_alpha=da)
        return run

    def single_step_da():
        pc.select_mesh_by_timestep(0)
        for i, c in enumerate(cams):
            o = render(c, pc, Pipe, bg, depth_alpha=True)
            loss_of(o["render"], gts_f[i], mask[i], o["alpha"], o["depth"]).backward()

    def views_step(da):
        def run():
            pc.select_mesh_by_timestep(0)
            for j, g in enumerate(groups):
                sl = slice(j * K, (j + 1) * K)
                o = render_views_train(g, pc, Pipe, bg, depth_alpha=da)
                # the mean over the K views of the per-view loss: the same objective as the K single-view steps
                loss = loss_of(o["render"], gts_f[sl], mask[sl], o.get("alpha"), o.get("depth")) * K
                loss.backward()
        return run

    return {"single_display_da": single_display_da, "views_da": views_forward(True), "views": views_forward(False),
            "single_step_da": single_step_da, "views_step_da": views_step(True), "views_step": views_step(False)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the lines to this file")
    args = ap.parse_args()
    info = gpu_info()
    lines = []
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p", 100_000, 1920, 1080)):
        pc, cams, gts = setting(P, W, H)
        for K in (4, 16):
            a = arms(pc, cams, gts, K)
            for fn in a.values():   # warm-up pass (allocator, hints)
                fn()
            torch.cuda.synchronize()
            ms = {k: [] for k in a}
            for _ in range(args.passes):   # the arms alternate pass by pass
                for k, fn in a.items():
                    ms[k] += timed(fn, passes=1)
            views = len(cams)
            for arm in a:
                t = sorted(ms[arm])
                rec = dict(setting=name, P=P, W=W, H=H, K=K, arm=arm, views_per_pass=views,
                           ms_per_view_median=t[len(t) // 2] / views, ms_per_view_min=t[0] / views,
                           ms_per_view_max=t[-1] / views, passes=len(t), **info)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
            del a
        del pc
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
