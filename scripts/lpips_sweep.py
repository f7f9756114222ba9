"""Per-view cost of the LPIPS distance (AlexNet as train.py's training_report scores it, VGG-16 as metrics.py does) ->
one JSON line per (network, setting, arm) on stdout, and per-layer lines (appended to profiles/h100/lpips.jsonl):

  reference   lpipsPyTorch's computation restated in torch (tests/lpips_oracle.py: z-score, F.conv2d + relu with
              cuDNN's defaults -- TF32 on an H100 -- max_pool2d, the normalised head), weights on the device once,
              warmed up, on pre-rendered float views: the LPIPS alone
  eager       lpips() (gab200_lpips) on the same pre-rendered views
  graph       GraphedEval over the views with and without lpips=: render + metrics (+ LPIPS) per replay; the
              difference is what LPIPS adds to an evaluation replay

Settings: the demo (550x802, 89,021 splats) and 100k splats at 1920x1080 (eval_sweep.py's synthetic FLAME avatar),
16 views per pass, the median of 3 passes after a warm-up pass.  Seeded weights (the cost does not depend on their
values).  Per layer, in a separate profiled pass: each lpips_conv_kernel launch's device time (torch.profiler) against
the reference's F.conv2d + relu of the same layer on the same two images (CUDA events over 10 launches), and the
achieved TFLOP/s of both from the MAC counts (2 FLOP per MAC, both images).  Every line carries the card and its power
limit, read in the same run."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..")))
sys.path.insert(0, HERE)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import eval_sweep as E  # noqa: E402
from gaussianavatars_b200.graph import GraphedEval  # noqa: E402
from gaussianavatars_b200.lpips import LpipsNet, lpips  # noqa: E402
from gaussianavatars_b200.renderer import render  # noqa: E402
from tests import lpips_oracle as ol  # noqa: E402

dev = E.dev
TF32_DATASHEET = 495.0   # H100 SXM dense TF32, NVIDIA data sheet (700 W)


def layer_macs(name, H, W):
    """[(module, Cin, Cout, k, Ho, Wo, MACs of both images)] of every convolution."""
    out = []
    spec = ol.NETS[name]
    for (mod, cin, cout, k, pool, _), (_, s, p, _, _) in zip(spec["convs"], ol.conv_specs(name)):
        H, W = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        out.append((mod, cin, cout, k, H, W, 2 * H * W * cout * cin * k * k))
        if pool:
            H, W = (H - spec["pool"]) // 2 + 1, (W - spec["pool"]) // 2 + 1
    return out


def main():
    info = E.gpu_info()
    for setting, P, W, H in (("demo", 89_021, 550, 802), ("1080p_100k", 100_000, 1920, 1080)):
        pc, views, gts, bg = E.setting(P, W, H)
        views, gts = views[:16], gts[:16]
        n = len(views)
        with torch.no_grad():
            imgs = []
            for c, t in views:
                pc.select_mesh_by_timestep(t)
                imgs.append(render(c, pc, Pipe, bg)["render"].clone())
        for name in ("alex", "vgg"):
            feats, lin = ol.seeded_weights(name, ol.SEED[name])
            net = LpipsNet(name, feats, lin, dev)
            fd = {k: v.to(dev) for k, v in feats.items()}
            ld = {k: v.to(dev) for k, v in lin.items()}
            res = {}

            def reference():
                total = 0.0
                with torch.no_grad():
                    for im, gt in zip(imgs, gts):
                        x, y = im.clamp(0, 1)[None], (gt.float() / 255)[None]
                        total += ol.lpips(x, y, name, fd, ld)[0].double()
                res["reference"] = float(total / n)

            def eager():
                res["eager"] = float(torch.stack([lpips(im, gt, net) for im, gt in zip(imgs, gts)]).double().mean())

            evs = {}
            for arm, lp in (("graph_lpips", net), ("graph_plain", None)):
                evs[arm] = GraphedEval(pc, W, H, bg, views=n, warm_cameras=[c for c, _ in views],
                                       warm_timesteps=(0, 2, 4, 6), lpips=lp)

            def graph(arm):
                ev = evs[arm]
                ev.reset()
                for i, ((c, t), gt) in enumerate(zip(views, gts)):
                    ev.set_inputs(camera=c, timestep=t, gt_u8=gt, view=i)
                    ev.run()
                s = ev.scores()
                res[arm] = s.get("lpips", float("nan"))

            times = {}
            for arm, fn in (("reference", reference), ("eager", eager), ("graph_lpips", lambda: graph("graph_lpips")),
                            ("graph_plain", lambda: graph("graph_plain"))):
                ms = E.timed(fn)
                times[arm] = ms[1] / n
                line = {"net": name, "setting": setting, "arm": arm, "splats": P, "W": W, "H": H,
                        "views_per_pass": n, "ms_per_view_median": round(ms[1] / n, 4),
                        "ms_per_view_best": round(ms[0] / n, 4), "passes": 3, "lpips_mean": res.get(arm), **info}
                print(json.dumps(line), flush=True)
            assert all(ev.captures == 1 and not ev.overflowed() for ev in evs.values())
            layers = layer_macs(name, H, W)
            gflop = sum(2 * m[-1] for m in layers) / 1e9
            print(json.dumps({"net": name, "setting": setting, "arm": "graph_difference", "W": W, "H": H,
                              "ms_per_view_lpips_in_graph": round(times["graph_lpips"] - times["graph_plain"], 4),
                              "gflop_per_pair": round(gflop, 2),
                              "achieved_tflops_eager": round(gflop / times["eager"], 1),
                              "achieved_tflops_reference": round(gflop / times["reference"], 1), **info}), flush=True)

            # per kernel, a separate profiled pass of eager calls
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for im, gt in zip(imgs[:4], gts[:4]):
                    lpips(im, gt, net)
                torch.cuda.synchronize()
            kern, convs = {}, []
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA and "lpips_" in e.name:
                    key = e.name.split("lpips_")[1].split("_kernel")[0]
                    kern.setdefault(key, []).append(e.device_time_total)
                    if key == "conv":
                        convs.append(e.device_time_total)
            per_call = {k: round(sum(v) / 4, 1) for k, v in kern.items()}
            nl = len(layers)
            x = torch.stack([imgs[0].clamp(0, 1), gts[0].double().div(255).float()])
            h = ol.z_score(x)
            for l, (mod, cin, cout, k, Ho, Wo, macs) in enumerate(layers):
                ours = sorted(convs[l::nl])[len(convs[l::nl]) // 2]
                _, s, p, pool, _ = ol.conv_specs(name)[l]
                w, b = fd[f"features.{mod}.weight"], fd[f"features.{mod}.bias"]
                f = lambda: F.relu(F.conv2d(h, w, b, stride=s, padding=p))  # noqa: E731
                for _ in range(3):
                    out = f()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(10):
                    out = f()
                e1.record()
                torch.cuda.synchronize()
                ref_us = e0.elapsed_time(e1) * 100.0
                print(json.dumps({"net": name, "setting": setting, "arm": "layer", "module": mod, "Cin": cin,
                                  "Cout": cout, "k": k, "Ho": Ho, "Wo": Wo, "gflop": round(2 * macs / 1e9, 3),
                                  "kernel_us": round(ours, 1), "cudnn_conv_relu_us": round(ref_us, 1),
                                  "kernel_tflops": round(2 * macs / ours / 1e6, 1),
                                  "cudnn_tflops": round(2 * macs / ref_us / 1e6, 1),
                                  "kernel_share_of_tf32_datasheet": round(2 * macs / ours / 1e6 / TF32_DATASHEET, 3),
                                  **info}), flush=True)
                h = F.max_pool2d(out, ol.NETS[name]["pool"], 2) if pool else out
            print(json.dumps({"net": name, "setting": setting, "arm": "kernels_us_per_call", "kernels": per_call,
                              **info}), flush=True)
            del evs, net
            torch.cuda.empty_cache()
        del pc
        torch.cuda.empty_cache()


Pipe = E.Pipe

if __name__ == "__main__":
    main()
