"""Per-view cost of scoring an avatar against its ground truth (l1, psnr, ssim per view, as train.py's training_report
and metrics.py do), three arms over the same views -> one JSON line per (setting, arm) on stdout (appended to
profiles/h100/eval.jsonl):

  reference   eager render() + torch.clamp + l1 / psnr / the conv2d SSIM written in torch (11x11 Gaussian window,
              grouped conv2d, zero padding), each view's three scalars accumulated as train.py accumulates them
  eager_cuda  eager render() + training.image_metrics (two launches)
  graph       GraphedEval: one replay per view (pose, render, metrics) and one synchronisation at the end

Views: 16 cameras with distinct fields of view x 4 FLAME timesteps = 64 views per pass; every arm runs 3 passes after
a warm-up pass and reports the median per-view time.  Renders are under no_grad in every arm.  Settings: the demo
(550x802, 89,021 splats) and 100k splats at 1920x1080, both with a synthetic FLAME head posed per view.  The metrics
kernels' own device time comes from torch.profiler over one pass of eager image_metrics calls.  Every line carries the
card and its power limit, read in the same run."""
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from gaussianavatars_b200 import image_metrics, synthetic as syn  # noqa: E402
from gaussianavatars_b200.flame import FlameLBS  # noqa: E402
from gaussianavatars_b200.graph import GraphedEval  # noqa: E402
from gaussianavatars_b200.model import MeshBoundGaussians  # noqa: E402
from gaussianavatars_b200.renderer import render  # noqa: E402

dev = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_W": float(q[1])} if len(q) == 2 else {"gpu": torch.cuda.get_device_name(dev)}


def rig(W, H, n=16):
    cams = []
    for i in range(n):
        orb = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=-50 + 100 * i / (n - 1),
                               elevation_deg=6 * math.sin(i))
        f = 1.0 + 0.08 * (2 * i / (n - 1) - 1)
        cams.append(syn.look_at_camera(W, H, math.degrees(orb.FoVx) * f, math.degrees(orb.FoVy) * f,
                                       w2c=orb.world_view_transform.T.numpy()).to(dev))
    return cams


def ssim_torch(img1, img2):
    """SSIM as the reference defines it (11x11 Gaussian window, sigma 1.5, grouped conv2d, padding 5), in torch."""
    g = torch.tensor([math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)])
    g = g / g.sum()
    w = (g[:, None] @ g[None, :]).expand(3, 1, 11, 11).contiguous().to(img1)
    conv = lambda a: F.conv2d(a, w, padding=5, groups=3)  # noqa: E731
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu12 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(img1 * img1) - mu1_sq, conv(img2 * img2) - mu2_sq, conv(img1 * img2) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))).mean()


def setting(P, W, H, T=8):
    a = syn.flame_like_assets(0)
    fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0]).items()
          if k != "dynamic_offset"}
    lbs = lambda: FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"],  # noqa: E731
                                       list(a["parents"]), a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"],
                                       device=dev)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, None, None, device=dev, flame=lbs(), flame_param=fp)
    g = torch.Generator().manual_seed(11)
    params2 = dict(params)   # the ground-truth avatar: the same head with perturbed colours
    params2["_features_dc"] = params["_features_dc"] + 0.25 * torch.randn(params["_features_dc"].shape, generator=g)
    truth = MeshBoundGaussians(params2, 3, None, None, device=dev, flame=lbs(), flame_param=fp)
    cams = rig(W, H)
    views = [(c, t) for t in (0, 2, 4, 6) for c in cams]
    bg = torch.ones(3, device=dev)
    gts = []
    with torch.no_grad():
        for c, t in views:
            truth.select_mesh_by_timestep(t)
            im = render(c, truth, Pipe, bg)["render"]
            gts.append(im.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).contiguous())
    return pc, views, gts, bg


def timed(fn, passes=3):
    fn()   # warm-up pass
    torch.cuda.synchronize()
    ms = []
    for _ in range(passes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return sorted(ms)


def main():
    out = []
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p_100k", 100_000, 1920, 1080)):
        pc, views, gts, bg = setting(P, W, H)
        gts_f = [g.float() / 255 for g in gts]
        n = len(views)
        res = {}

        def reference():
            l1_t = psnr_t = ssim_t = 0.0
            with torch.no_grad():
                for (c, t), gt in zip(views, gts_f):
                    pc.select_mesh_by_timestep(t)
                    image = torch.clamp(render(c, pc, Pipe, bg)["render"], 0.0, 1.0)
                    gt_image = torch.clamp(gt, 0.0, 1.0)
                    l1_t += (image - gt_image).abs().mean().double()
                    mse = ((image - gt_image) ** 2).view(3, -1).mean(1, keepdim=True)
                    psnr_t += (20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double()
                    ssim_t += ssim_torch(image[None], gt_image[None]).double()
            res["reference"] = torch.stack([l1_t, psnr_t, ssim_t]) / n

        def eager_cuda():
            recs = []
            with torch.no_grad():
                for (c, t), gt in zip(views, gts):
                    pc.select_mesh_by_timestep(t)
                    recs.append(image_metrics(render(c, pc, Pipe, bg)["render"], gt))
            res["eager_cuda"] = torch.stack(recs).double().mean(0)

        ev = GraphedEval(pc, W, H, bg, views=n, warm_cameras=[c for c, _ in views[:16]], warm_timesteps=(0, 2, 4, 6))

        def graph():
            ev.reset()
            for i, ((c, t), gt) in enumerate(zip(views, gts)):
                ev.set_inputs(camera=c, timestep=t, gt_u8=gt, view=i)
                ev.run()
            res["graph"] = ev.scores()

        for arm, fn in (("reference", reference), ("eager_cuda", eager_cuda), ("graph", graph)):
            ms = timed(fn)
            out.append({"setting": name, "arm": arm, "splats": P, "W": W, "H": H, "views_per_pass": n,
                        "ms_per_view_median": round(ms[1] / n, 4), "ms_per_view_best": round(ms[0] / n, 4),
                        "passes": 3, "runs": 1})
        assert not ev.overflowed() and ev.captures == 1
        s = res["graph"]
        agree = {"reference": [round(float(v), 5) for v in res["reference"]],
                 "eager_cuda": [round(float(res["eager_cuda"][i]), 5) for i in (0, 1, 3)],
                 "graph": [round(s["l1"], 5), round(s["psnr"], 5), round(s["ssim"], 5)]}

        # the metrics kernels' device time: one pass of eager image_metrics calls on prepared renders
        with torch.no_grad():
            imgs = []
            for (c, t) in views:
                pc.select_mesh_by_timestep(t)
                imgs.append(render(c, pc, Pipe, bg)["render"].clone())
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for im, gt in zip(imgs, gts):
                image_metrics(im, gt)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if "metrics_" in e.key:
                kern["tile" if "tile" in e.key else "finalize"] = round(e.device_time_total / max(e.count, 1), 2)
        alg = 3 * H * W * 4 + 3 * H * W   # float render + uint8 ground truth
        for line in out[-3:]:
            line.update({"metric_means_l1_psnr_ssim": agree[line["arm"]],
                         "metrics_kernel_us": kern, "metrics_algorithmic_bytes": alg, **gpu_info()})
            print(json.dumps(line), flush=True)
        del ev, pc
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
