"""PNG files read on the device (gaussianavatars_b200.png.decode_png, FrameStore.add_png): one JSON line per
measurement to stdout and to --out (profiles/h100/png_decode.jsonl).  Every file is held in memory: no disk time.

  gpu       the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  decode    decode_png of F = 16, 64, 256, 1024 files: 802x550 RGBA synthetic avatar frames written by PIL at level 6
            (the capture's frames), 1920x1080 RGB display frames written by PIL at level 6 and by encode_png (render.py's
            files).  16 different frames, repeated.  After warm-up: CUDA events around the call (upload and the two
            kernels), the host time of the whole call (chunk walk, packing, launch, the status read), files/s of
            each; and PIL's decode of the same files in a ThreadPoolExecutor(os.cpu_count()) (PIL releases the GIL
            while it inflates)
  store     a FrameStore filled with 1024 demo frames: PIL pool + add_rgba against add_png at several batch sizes
  kernels   png_inflate_kernel and png_unfilter_kernel's share of one F = 64 decode of each kind (torch.profiler, a run
            of its own)

    python scripts/png_decode_sweep.py --out profiles/h100/png_decode.jsonl
"""
from __future__ import annotations

import argparse
import io
import json
import math
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


BATCHES = (16, 64, 256, 1024)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"kind": "gpu", "name": name, "power_limit": power, "max_sm_clock": clock, "cpu_count": os.cpu_count(),
            "torch": torch.__version__, "cuda": torch.version.cuda}


@torch.no_grad()
def frames(P, W, H, dev, n=16):
    """n display frames (RGB) and their alpha planes (RGBA) of the synthetic avatar, orbiting."""
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render_display
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=dev)
    pc.select_mesh_by_timestep(0)
    rgb, rgba = [], []
    for i in range(n):
        cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=-40 + 80 * i / (n - 1),
                               elevation_deg=5.0 * math.sin(i))
        out = render_display(cam, pc, Pipe, torch.ones(3, device=dev), depth_alpha=True)
        a = (out["alpha"][0] * 255 + 0.5).clamp(0, 255).to(torch.uint8)
        rgb.append(out["display_u8"].contiguous())
        rgba.append(torch.cat([out["display_u8"], a[..., None]], 2).contiguous())
    return rgb, rgba


def pil_files(imgs, level=6):
    from PIL import Image
    out = []
    for t in imgs:
        buf = io.BytesIO()
        Image.fromarray(t.cpu().numpy()).save(buf, format="PNG", compress_level=level)
        out.append(buf.getvalue())
    return out


def pil_decode(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"))


def time_device(files, channels, dev, reps):
    from gaussianavatars_b200 import decode_png
    for _ in range(2):
        decode_png(files, channels, dev)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dev_ms, host_ms = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        ev[0].record()
        out = decode_png(files, channels, dev)
        ev[1].record()
        ev[1].synchronize()
        host_ms.append(1e3 * (time.perf_counter() - t0))
        dev_ms.append(ev[0].elapsed_time(ev[1]))
        del out
    return float(np.median(dev_ms)), float(np.median(host_ms))


def time_pool(files, reps):
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        list(ex.map(pil_decode, files[:32]))
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            list(ex.map(pil_decode, files))
            ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def decode_lines(kind, files16, W, H, channels, dev):
    out = []
    for F in BATCHES:
        files = [files16[i % len(files16)] for i in range(F)]
        reps = 5 if F <= 256 else 3
        dev_ms, host_ms = time_device(files, channels, dev, reps)
        pool_ms = time_pool(files, reps)
        torch.cuda.empty_cache()
        out.append({"kind": "decode", "files": kind, "W": W, "H": H, "channels": channels, "F": F,
                    "mean_file_bytes": int(np.mean([len(f) for f in files])),
                    "device_ms": round(dev_ms, 3), "host_call_ms": round(host_ms, 3),
                    "device_files_per_s": round(F / host_ms * 1e3, 1), "pil_pool_ms": round(pool_ms, 3),
                    "pil_pool_files_per_s": round(F / pool_ms * 1e3, 1), "reps": reps,
                    "device_over_pool": round(pool_ms / host_ms, 3)})
        print(json.dumps(out[-1]), flush=True)
    return out


def store_lines(files16, W, H, dev):
    from gaussianavatars_b200 import FrameStore
    files = [files16[i % len(files16)] for i in range(1024)]
    out = []

    def pil_fill():
        s = FrameStore(W, H, [1.0, 1.0, 1.0], dev)
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            for i in range(0, 1024, 64):
                rgba = np.stack(list(ex.map(pil_decode, files[i:i + 64])))
                s.add_rgba(torch.from_numpy(rgba))
        torch.cuda.synchronize()
        return s

    def png_fill(batch):
        s = FrameStore(W, H, [1.0, 1.0, 1.0], dev)
        s.add_png(files, batch=batch)
        torch.cuda.synchronize()
        return s

    arms = [("pil_pool+add_rgba", pil_fill)] + [(f"add_png(batch={b})", lambda b=b: png_fill(b))
                                                for b in (16, 64, 256)]
    ref = None
    for name, fn in arms:
        fn()   # warm-up
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            s = fn()
            ts.append(time.perf_counter() - t0)
        gt, mask = s.decode(list(range(0, 1024, 97)))
        same = None if ref is None else bool(torch.equal(gt, ref[0]) and torch.equal(mask, ref[1]) and
                                             s.nbytes == ref[2])
        if ref is None:
            ref = (gt, mask, s.nbytes)
        out.append({"kind": "store", "arm": name, "frames": 1024, "W": W, "H": H, "s": round(float(np.median(ts)), 3),
                    "frames_per_s": round(1024 / float(np.median(ts)), 1), "same_as_pil": same})
        print(json.dumps(out[-1]), flush=True)
        del s
        torch.cuda.empty_cache()
    return out


def kernel_lines(sets, dev, trace_dir):
    from torch.profiler import ProfilerActivity, profile
    from gaussianavatars_b200 import decode_png
    out = []
    for kind, files16, channels in sets:
        files = [files16[i % len(files16)] for i in range(64)]
        decode_png(files, channels, dev)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                decode_png(files, channels, dev)
            torch.cuda.synchronize()
        if trace_dir:
            prof.export_chrome_trace(os.path.join(trace_dir, f"png_decode_{kind}.pt.trace.json"))
        tot = {}
        for e in prof.key_averages():
            if "png_inflate_kernel" in e.key or "png_unfilter_kernel" in e.key:
                k = "inflate" if "inflate" in e.key else "unfilter"
                tot[k] = tot.get(k, 0.0) + e.device_time_total / 1e3 / 3
        out.append({"kind": "kernels", "files": kind, "F": 64, "inflate_ms": round(tot.get("inflate", 0.0), 3),
                    "unfilter_ms": round(tot.get("unfilter", 0.0), 3)})
        print(json.dumps(out[-1]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the sweep measures the device: it needs a GPU"
    dev = torch.device("cuda:0")
    from gaussianavatars_b200 import encode_png
    lines = [gpu_info()]
    print(json.dumps(lines[0]), flush=True)
    _, demo_rgba = frames(89_000, 802, 550, dev)
    hd_rgb, _ = frames(100_000, 1920, 1080, dev)
    demo = pil_files(demo_rgba)
    hd_pil = pil_files(hd_rgb)
    hd_enc = [encode_png(t) for t in hd_rgb]
    for kind, files, W, H, ch in (("demo_rgba_pil6", demo, 802, 550, 4), ("1080p_rgb_pil6", hd_pil, 1920, 1080, 3),
                                  ("1080p_rgb_encode_png", hd_enc, 1920, 1080, 3)):
        lines += decode_lines(kind, files, W, H, ch, dev)
    lines += store_lines(demo, 802, 550, dev)
    lines += kernel_lines((("demo_rgba_pil6", demo, 4), ("1080p_rgb_pil6", hd_pil, 3),
                           ("1080p_rgb_encode_png", hd_enc, 3)), dev, args.trace_dir)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
