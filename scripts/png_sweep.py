"""PNG files on the device (gaussianavatars_b200.png, GraphedRender(png=True)): one JSON line per measurement to
stdout and to --out (profiles/h100/png.jsonl).

  gpu          the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  encode       gab200_png_encode alone on display frames of the synthetic avatar (802x550 with 89k splats, 1920x1080
               with 100k), K = 1 and K = 16 views per launch: CUDA events around --launches launches after warm-up,
               ms per view; the bytes of each file against PIL's compress_level 6 (render.py's default) and 1, and
               PIL's host encode time for the same frames
  kernels      the six kernels' share of one 1920x1080 encode at K = 1 and K = 16 (torch.profiler, a run of its own)
  loop         render.py's loop: a GraphedRender replay per frame, the file bytes in host memory -- png=True and
               host_png(i - 1) against host_frame(i - 1) + PIL save (compress_level 6): frames per second

    python scripts/png_sweep.py --out profiles/h100/png.jsonl
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


SIZES = ((802, 550, 89_000), (1920, 1080, 100_000))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"kind": "gpu", "name": name, "power_limit": power, "max_sm_clock": clock,
            "torch": torch.__version__, "cuda": torch.version.cuda}


def avatar(P, W, H, dev):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=dev)
    pc.select_mesh_by_timestep(0)
    cams = [syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=-40 + 80 * i / 15,
                             elevation_deg=5.0 * math.sin(i)) for i in range(16)]
    return pc, cams


@torch.no_grad()
def displays(pc, cams, dev):
    from gaussianavatars_b200.renderer import render_display
    return torch.stack([render_display(c, pc, Pipe, torch.ones(3, device=dev))["display_u8"] for c in cams])


def encode_lines(pc, cams, W, H, P, dev, launches):
    from PIL import Image
    from gaussianavatars_b200 import png as PNG
    frames = displays(pc, cams, dev).contiguous()
    out = []
    for K in (1, 16):
        u8 = frames[:K].contiguous()
        buf = torch.empty((K, PNG.slot_stride(W, H)), dtype=torch.uint8, device=dev)
        lens = torch.empty(K, dtype=torch.int64, device=dev)
        sc = PNG.scratch(K, H, W, dev)
        for _ in range(5):
            PNG.launch_encode(u8, sc, buf, lens)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            PNG.launch_encode(u8, sc, buf, lens)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / launches
        out.append({"kind": "encode", "width": W, "height": H, "splats": P, "views": K, "launches": launches,
                    "ms_per_launch": ms, "ms_per_view": ms / K})
    files = PNG.encode_png(frames)
    raw = W * H * 3
    for k in range(4):
        img = frames[k].cpu().numpy()
        row = {"kind": "bytes", "width": W, "height": H, "splats": P, "view": k, "raw": raw, "device": len(files[k])}
        for level in (6, 1):
            t0 = time.perf_counter()
            bio = io.BytesIO()
            Image.fromarray(img).save(bio, format="PNG", compress_level=level)
            row[f"pil{level}"] = bio.tell()
            row[f"pil{level}_host_ms"] = (time.perf_counter() - t0) * 1e3
        row["ratio_device_raw"] = row["device"] / raw
        row["ratio_device_pil6"] = row["device"] / row["pil6"]
        row["ratio_device_pil1"] = row["device"] / row["pil1"]
        out.append(row)
    return out, frames


def kernel_lines(frames, W, H, dev):
    from torch.profiler import ProfilerActivity, profile
    from gaussianavatars_b200 import png as PNG
    out = []
    for K in (1, 16):
        u8 = frames[:K].contiguous()
        buf = torch.empty((K, PNG.slot_stride(W, H)), dtype=torch.uint8, device=dev)
        lens = torch.empty(K, dtype=torch.int64, device=dev)
        sc = PNG.scratch(K, H, W, dev)
        PNG.launch_encode(u8, sc, buf, lens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                PNG.launch_encode(u8, sc, buf, lens)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            for name in ("png_filter_kernel", "png_lz_kernel", "png_offsets_kernel", "png_pack_kernel",
                         "png_assemble_kernel", "png_finish_kernel"):
                if name in e.key:
                    t = getattr(e, "device_time_total", None)
                    t = e.cuda_time_total if t is None else t
                    per[name] = per.get(name, 0.0) + t / 1e3 / 10
        out.append({"kind": "kernels", "width": W, "height": H, "views": K, "ms_per_launch": per})
    return out


def loop_lines(pc, cams, W, H, P, frames_n, dev):
    from PIL import Image
    from gaussianavatars_b200.graph import GraphedRender
    out = []
    bg = torch.ones(3)
    for mode in ("png", "pil"):
        view = GraphedRender(pc, W, H, bg, outputs="u8", host_slots=2, png=mode == "png", warm_cameras=cams)
        total = 0

        def consume(i):
            nonlocal total
            if mode == "png":
                total += len(view.host_png(i))
            else:
                bio = io.BytesIO()
                Image.fromarray(view.host_frame(i).numpy()).save(bio, format="PNG", compress_level=6)
                total += bio.tell()

        for i in range(4):   # capture and warm-up
            view.set_inputs(camera=cams[i % 16])
            view.run(check=True)
        torch.cuda.synchronize()
        base = view.replays
        total = 0
        t0 = time.perf_counter()
        for i in range(frames_n):
            view.set_inputs(camera=cams[i % 16])
            view.run()
            if i >= 1:
                consume(base + i - 1)
        consume(base + frames_n - 1)
        sec = time.perf_counter() - t0
        assert not view.overflowed()
        out.append({"kind": "loop", "mode": mode, "width": W, "height": H, "splats": P, "frames": frames_n,
                    "frames_per_s": frames_n / sec, "mean_file_bytes": total / frames_n, "captures": view.captures})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--loop-frames", type=int, default=64)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the sweep measures on a GPU"
    dev = torch.device("cuda:0")
    lines = [gpu_info()]
    for W, H, P in SIZES:
        pc, cams = avatar(P, W, H, dev)
        enc, frames = encode_lines(pc, cams, W, H, P, dev, args.launches)
        lines += enc
        if W == 1920:
            lines += kernel_lines(frames, W, H, dev)
        lines += loop_lines(pc, cams, W, H, P, args.loop_frames, dev)
    sink = open(args.out, "w") if args.out else None
    for line in lines:
        s = json.dumps(line)
        print(s)
        if sink:
            sink.write(s + "\n")
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
