"""What training on the capture's RGBA frames costs -> one JSON line per measurement on stdout
(profiles/h100/rgba_mask.jsonl):

  iteration   per-view time of the captured training iteration (GraphedFrame, FLAME pose + render + photometric loss +
              regularisers + backward + densification statistics + capturable Adam), three arms:
                (a) gt_u8      the ground truth uploaded as the (3,H,W) uint8 composite
                (b) rgba       rgba=True: the (H,W,4) frame, composited inside the graph
                (c) rgba_mask  rgba=True, lambda_mask=0.1: also the alpha plane and the mask term
              A pass is 16 cameras x 2 FLAME timesteps = 32 views, K views per replay; the arms alternate pass by
              pass, 5 passes each after a warm-up pass; the median and the spread are reported.
  composite   gab200_composite_rgba alone: CUDA events around 200 launches, per view, and the bytes it moves
              (4 read + 4 written per pixel) over that time.
  host        the loader's per-pixel float64 composite restated in numpy, against decoding the PNG alone (PIL,
              in-memory PNG of a synthetic RGBA frame), on this machine's CPU, median of 5.

Settings: the demo (550x802, 89,021 splats) and 100k splats at 1920x1080, K in {1, 16}.  Every line carries the card,
its power limit and its SM clock, read in the same run."""
import io
import json
import os
import sys
import time

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import gaussianavatars_b200 as g  # noqa: E402
from gaussianavatars_b200.graph import GraphedFrame  # noqa: E402
from gaussianavatars_b200.training import launch_composite_rgba  # noqa: E402
from scripts.train_views_sweep import gpu_info, setting, timed  # noqa: E402

dev = torch.device("cuda:0")
STEPS = (0, 5)
VIEWS = 16 * len(STEPS)
PASSES = 5
ARMS = {"gt_u8": {}, "rgba": {"rgba": True}, "rgba_mask": {"rgba": True, "lambda_mask": 0.1}}


def rgba_frames(n, H, W, seed=3):
    """n synthetic RGBA captures: random colours, an opaque head-like ellipse, transparent outside, a soft edge."""
    gen = torch.Generator().manual_seed(seed)
    rgba = torch.randint(0, 256, (n, H, W, 4), generator=gen, dtype=torch.uint8)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    r = (xx / 0.5) ** 2 + (yy / 0.7) ** 2
    rgba[..., 3] = (255 * (1.2 - r).clamp(0, 0.2) / 0.2).to(torch.uint8)
    return rgba


def iteration_arms(pc, opt, cams, rgba, W, H, K):
    bg = torch.ones(3, device=dev)
    gts = g.composite_rgba(rgba, bg)[0]
    groups = [cams[i:i + K] for i in range(0, 16, K)]
    warm = groups if K > 1 else cams
    fns, frames = {}, []
    for arm, kw in ARMS.items():
        fr = GraphedFrame(pc, W, H, 1.0, 1.0, torch.ones(3), loss="photometric", regularizers={}, optimizer=opt,
                          densify_stats=True, per_camera_fov=True, views_per_replay=K, warm_cameras=warm, **kw)
        frames.append(fr)

        def run(fr=fr, rgba_in=bool(kw)):
            for t in STEPS:
                for j, grp in enumerate(groups):
                    sl = slice(j * K, (j + 1) * K)
                    gt = dict(gt_rgba=rgba[sl] if K > 1 else rgba[j]) if rgba_in else \
                        dict(gt_u8=gts[sl] if K > 1 else gts[j])
                    if K > 1:
                        fr.set_inputs(cameras=grp, timestep=t, **gt)
                    else:
                        fr.set_inputs(camera=grp[0], timestep=t, **gt)
                    fr.run()
        fns[arm] = run
    return fns, frames


def composite_lines(name, H, W, info):
    out = []
    bg = torch.ones(3, device=dev)
    for K in (1, 16):
        rgba = rgba_frames(K, H, W).to(dev)
        gt = torch.empty((K, 3, H, W), dtype=torch.uint8, device=dev)
        mask = torch.empty((K, 1, H, W), dtype=torch.uint8, device=dev)
        for _ in range(10):
            launch_composite_rgba(rgba, bg, gt, mask)
        n = 200

        def many():
            for _ in range(n):
                launch_composite_rgba(rgba, bg, gt, mask)
        ms = sorted(timed(many) for _ in range(5))
        us = ms[2] * 1e3 / n
        out.append(dict(setting=name, W=W, H=H, K=K, arm="composite", launches=n, us_per_launch_median=round(us, 3),
                        us_per_view_median=round(us / K, 3), us_per_launch_min=round(ms[0] * 1e3 / n, 3),
                        bytes_per_launch=8 * K * H * W, GB_per_s=round(8 * K * H * W / (us * 1e-6) / 1e9, 1), **info))
    return out


def host_line(name, H, W, info):
    from PIL import Image
    frame = rgba_frames(1, H, W)[0].numpy()
    buf = io.BytesIO()
    Image.fromarray(frame, "RGBA").save(buf, format="PNG")
    png = buf.getvalue()
    bg = np.array([1, 1, 1])

    def decode():
        return np.asarray(Image.open(io.BytesIO(png)).convert("RGBA"))

    def composite(im):
        norm = im / 255.0
        arr = norm[:, :, :3] * norm[:, :, 3:4] + bg * (1 - norm[:, :, 3:4])
        return np.array(arr * 255.0).astype(np.int8)

    def med(fn, *a):
        ts = []
        for _ in range(5):
            t0 = time.perf_counter()
            fn(*a)
            ts.append(time.perf_counter() - t0)
        return sorted(ts)[2] * 1e3
    im = decode()
    return dict(setting=name, W=W, H=H, arm="host", png_bytes=len(png), decode_ms_median=round(med(decode), 2),
                composite64_ms_median=round(med(composite, im), 2), cpu_count=os.cpu_count(), **info)


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p", 100_000, 1920, 1080)):
        pc, opt, cams, _ = setting(P, W, H)
        rgba = rgba_frames(16, H, W).to(dev)
        for K in (1, 16):
            fns, frames = iteration_arms(pc, opt, cams, rgba, W, H, K)
            for fn in fns.values():   # warm-up pass (captures)
                fn()
            torch.cuda.synchronize()
            ms = {k: [] for k in fns}
            for _ in range(PASSES):
                for k, fn in fns.items():
                    ms[k].append(timed(fn))
            overflow = any(f.overflowed() for f in frames)
            for arm, v in ms.items():
                v = sorted(v)
                emit({"setting": name, "splats": P, "W": W, "H": H, "K": K, "arm": arm, "views_per_pass": VIEWS,
                      "ms_per_view_median": round(v[len(v) // 2] / VIEWS, 4), "ms_per_view_min": round(v[0] / VIEWS, 4),
                      "ms_per_view_max": round(v[-1] / VIEWS, 4), "passes": len(v), "overflow": overflow,
                      "captures": [f.captures for f in frames], **info})
            del fns, frames
            torch.cuda.empty_cache()
        for rec in composite_lines(name, H, W, info):
            emit(rec)
        emit(host_line(name, H, W, info))
        del pc, opt, rgba
        torch.cuda.empty_cache()
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
