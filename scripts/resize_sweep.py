"""The loader's resize on the device (FrameStore.add_png(resize=True), gaussianavatars_b200.resize): one JSON line per
measurement to stdout and to --out (profiles/h100/resize.jsonl).  Every file is held in memory: no disk time.

  gpu      the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  store    64 RGBA capture frames (16 different synthetic avatar frames written by PIL at level 6, repeated) put into a
           FrameStore at the reference's --resolution -1 size: 3208x2200 -> 1600x1097 (full-resolution NeRSemble) and
           1920x1080 -> 1600x900.  add_png(resize=True) against PIL in a ThreadPoolExecutor(8) doing the same work per
           file (open, convert("RGBA"), the loader's float64 composite, resize of the "RGB" image and of the alpha as
           "L") followed by add(gt, mask).  Warm-up, then the median of 3 fills, each ending in a synchronise; the two
           stores' frames are compared byte for byte
  kernels  gab200_resize_u8 of the composited frames (3 colour planes + the mask plane per frame, F = 64), preallocated
           scratch: CUDA events around 20 calls after warm-up -> us per frame; and each kernel's share from
           torch.profiler in a run of its own

    python scripts/resize_sweep.py --out profiles/h100/resize.jsonl
"""
from __future__ import annotations

import argparse
import io
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from png_decode_sweep import frames, gpu_info, pil_files  # noqa: E402

F = 64
THREADS = 8
SIZES = ((3208, 2200, 150_000), (1920, 1080, 100_000))   # capture W, H, splats of the synthetic frames
BG = [1.0, 1.0, 1.0]


def pil_frame(data, w, h):
    """(gt (3,h,w), mask (1,h,w)) of one file the way the reference's loader makes it, plus the alpha resized."""
    from PIL import Image
    rgba = np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"))
    n = rgba / 255.0
    arr = n[:, :, :3] * n[:, :, 3:4] + np.asarray(BG) * (1 - n[:, :, 3:4])
    c = np.array(arr * 255.0).astype(np.int8)
    img = Image.frombuffer("RGB", (rgba.shape[1], rgba.shape[0]), c.tobytes(), "raw", "RGB", 0, 1)
    gt = np.asarray(img.resize((w, h))).transpose(2, 0, 1)
    mask = np.asarray(Image.fromarray(rgba[..., 3], "L").resize((w, h)))[None]
    return gt, mask


def store_lines(files, W, H, w, h, dev):
    from gaussianavatars_b200 import FrameStore
    out = []

    def pil_fill():
        s = FrameStore(w, h, BG, dev)
        with ThreadPoolExecutor(THREADS) as ex:
            for i in range(0, len(files), 16):
                res = list(ex.map(lambda d: pil_frame(d, w, h), files[i:i + 16]))
                s.add(torch.from_numpy(np.stack([r[0] for r in res])), torch.from_numpy(np.stack([r[1] for r in res])))
        torch.cuda.synchronize()
        return s

    def png_fill():
        s = FrameStore(w, h, BG, dev)
        s.add_png(files, resize=True)
        torch.cuda.synchronize()
        return s

    ref = None
    for name, fn in (("pil_pool+add", pil_fill), ("add_png(resize=True)", png_fill)):
        fn()   # warm-up
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            s = fn()
            ts.append(time.perf_counter() - t0)
        gt, mask = s.decode(list(range(0, len(files), 7)))
        same = None if ref is None else bool(torch.equal(gt, ref[0]) and torch.equal(mask, ref[1]))
        if ref is None:
            ref = (gt, mask)
        med = float(np.median(ts))
        out.append({"kind": "store", "arm": name, "frames": len(files), "W": W, "H": H, "w": w, "h": h,
                    "s": round(med, 3), "frames_per_s": round(len(files) / med, 1), "same_as_pil": same})
        del s
        torch.cuda.empty_cache()
    out[0]["threads"] = THREADS
    out[1]["device_over_pool"] = round(out[1]["frames_per_s"] / out[0]["frames_per_s"], 3)
    for line in out:
        print(json.dumps(line), flush=True)
    return out


def kernel_lines(files, W, H, w, h, dev):
    from torch.profiler import ProfilerActivity, profile
    from gaussianavatars_b200 import composite_rgba, decode_png
    from gaussianavatars_b200.resize import launch_resize, scratch_bytes
    rgba = decode_png(files, 4, dev)
    gt, mask = composite_rgba(rgba, BG)
    del rgba
    planes = torch.cat([gt, mask], 1).contiguous()                       # (F, 4, H, W)
    dst = torch.empty((F, 4, h, w), dtype=torch.uint8, device=dev)
    scratch = torch.empty(scratch_bytes(4 * F, H, W, h, w), dtype=torch.uint8, device=dev)
    for _ in range(3):
        launch_resize(planes, dst, scratch)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    n = 20
    ev[0].record()
    for _ in range(n):
        launch_resize(planes, dst, scratch)
    ev[1].record()
    ev[1].synchronize()
    ms = ev[0].elapsed_time(ev[1]) / n
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            launch_resize(planes, dst, scratch)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.key_averages():
        for k in ("resize_plan_kernel", "resize_horizontal_kernel", "resize_vertical_kernel"):
            if k in e.key:
                tot[k] = tot.get(k, 0.0) + e.device_time_total / 3 / F
    bytes_moved = F * 4 * (H * W + 2 * H * w + h * w)   # read src, write + read the intermediate, write dst
    line = {"kind": "kernels", "W": W, "H": H, "w": w, "h": h, "F": F, "planes_per_frame": 4,
            "ms_per_call": round(ms, 3), "us_per_frame": round(1e3 * ms / F, 2),
            "min_bytes_per_frame": bytes_moved // F, "achieved_GB_s": round(bytes_moved / (ms * 1e-3) / 1e9, 1),
            **{k.replace("_kernel", "_us_per_frame"): round(v, 2) for k, v in tot.items()}}
    print(json.dumps(line), flush=True)
    del planes, dst, scratch, gt, mask
    torch.cuda.empty_cache()
    return [line]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the sweep measures the device: it needs a GPU"
    dev = torch.device("cuda:0")
    from gaussianavatars_b200 import loader_size
    lines = [gpu_info()]
    print(json.dumps(lines[0]), flush=True)
    for W, H, P in SIZES:
        w, h = loader_size(W, H)
        _, rgba = frames(P, W, H, dev)
        files16 = pil_files(rgba)
        del rgba
        files = [files16[i % len(files16)] for i in range(F)]
        lines.append({"kind": "files", "W": W, "H": H, "w": w, "h": h, "distinct": len(files16),
                      "mean_file_bytes": int(np.mean([len(f) for f in files16]))})
        print(json.dumps(lines[-1]), flush=True)
        lines += store_lines(files, W, H, w, h, dev)
        lines += kernel_lines(files, W, H, w, h, dev)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
