"""The deblocking filter in the device H.264 encoder (VideoWriter(deblock=True), gab200_h264_encode_deblocked), off
against on: one JSON line per measurement to stdout and to --out (profiles/h100/video_deblock.jsonl).

  gpu     the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  size    bytes per frame and Y-PSNR of FFmpeg's decode against the source's Y plane, deblock off and on, qp 20, 26,
          32, 38, gop 1 and 25, on 64 display frames of the synthetic avatar (550x802 with 89k splats, 1920x1080 with
          100k) whose timestep advances under a fixed camera ("fixed") and under an orbiting one ("orbit")
  encode  ms per frame at gop 25 and qp 26, K = 1, 16, 64 frames per launch, eager and as a replayed CUDA graph, deblock
          off and on alternated in the same run (CUDA events around enough launches for 256 frames after warm-up)
  loop    render.py's loop with gop 25 and qp 26, deblock off and on: a GraphedRender replay per frame (fixed camera,
          timestep advancing) into a VideoWriter, the file on disk; frames per second

    python scripts/video_deblock_sweep.py --out profiles/h100/video_deblock.jsonl
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from png_sweep import avatar, gpu_info  # noqa: E402
from video_gop_sweep import clip  # noqa: E402
from video_sweep import decoded_y, source_y  # noqa: E402

SIZES = ((550, 802, 89_000), (1920, 1080, 100_000))
KS = (1, 16, 64)
QPS = (20, 26, 32, 38)
GOP = 25


def size_lines(frames, W, H, P, motion):
    from gaussianavatars_b200 import encode_video
    src = source_y(frames.cpu().numpy())
    out = []
    for qp in QPS:
        for gop in (1, GOP):
            for deblock in (False, True):
                data = encode_video(frames, qp=qp, gop=gop, deblock=deblock)
                ys = decoded_y(data, H, W)
                mse = np.mean([(y.astype(np.float64) - s) ** 2 for y, s in zip(ys, src)])
                out.append({"kind": "size", "width": W, "height": H, "splats": P, "motion": motion, "qp": qp,
                            "gop": gop, "deblock": deblock, "frames": len(frames), "decoded_frames": len(ys),
                            "bytes_per_frame": len(data) / len(frames),
                            "y_psnr_db": float(10 * np.log10(255 ** 2 / mse)) if mse else None})
    return out


def time_stream(frames, qp, gop, deblock, dev, graph, total_frames=256):
    from gaussianavatars_b200 import video as V
    K, H, W = V.check_frames(frames)
    st = V.state_buffer(H, W, dev)
    sc = V.deblocked_scratch(K, H, W, gop, dev) if deblock else V.scratch(K, H, W, dev)
    out = torch.empty((K, V.slot_stride(W, H, gop)), dtype=torch.uint8, device=dev)
    lens = torch.empty(K, dtype=torch.int64, device=dev)

    def launch():
        if deblock:
            V.launch_encode_deblocked(frames, qp, gop, st, sc, out, lens)
        else:
            V.launch_encode_stream(frames, qp, gop, st, sc, out, lens)

    n = max(4, total_frames // K)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            launch()
        g = None
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                launch()
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(n):
            if graph:
                g.replay()
            else:
                launch()
        e1.record(s)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (n * K)


def encode_lines(frames64, W, H, P, dev):
    out = []
    for K in KS:
        for graph in (False, True):
            for deblock in (False, True, False, True):          # alternated: each mode measured twice
                ms = time_stream(frames64[:K].contiguous(), 26, GOP, deblock, dev, graph)
                out.append({"kind": "encode", "width": W, "height": H, "splats": P, "gop": GOP, "qp": 26, "K": K,
                            "graph": graph, "deblock": deblock, "ms_per_frame": ms})
    return out


def loop_lines(pc, cams, W, H, P, frames_n, dev):
    from gaussianavatars_b200 import VideoWriter
    from gaussianavatars_b200.graph import GraphedRender
    poses = []                                     # the synthetic avatar has no FLAME head: posed vertices per step
    for t in range(8):
        pc.select_mesh_by_timestep(t)
        poses.append(pc.verts.detach().clone())
    pc.select_mesh_by_timestep(0)
    view = GraphedRender(pc, W, H, torch.ones(3), outputs="u8", warm_cameras=cams[:1])
    for i in range(4):
        view.set_inputs(camera=cams[0], verts=poses[i % 8])
        view.run(check=True)
    out = []
    for deblock in (False, True, False, True):
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "renders.mp4")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with VideoWriter(path, W, H, fps=25, qp=26, batch=16, gop=GOP, deblock=deblock) as vw:
                for i in range(frames_n):
                    view.set_inputs(camera=cams[0], verts=poses[i % 8])
                    view.run()
                    vw.add(view.display)
            sec = time.perf_counter() - t0
            size = os.path.getsize(path)
        out.append({"kind": "loop", "mode": "video", "width": W, "height": H, "splats": P, "frames": frames_n,
                    "qp": 26, "batch": 16, "gop": GOP, "deblock": deblock, "frames_per_s": frames_n / sec,
                    "file_bytes": size})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the lines to this file")
    ap.add_argument("--loop-frames", type=int, default=400)
    args = ap.parse_args()
    dev = torch.device("cuda")
    lines = []

    def emit(new):
        for ln in new:
            print(json.dumps(ln), flush=True)
        lines.extend(new)

    emit([gpu_info()])
    for W, H, P in SIZES:
        pc, cams = avatar(P, W, H, dev)
        fixed = clip(pc, cams, dev, orbit=False)
        emit(size_lines(fixed, W, H, P, "fixed"))
        emit(size_lines(clip(pc, cams, dev, orbit=True), W, H, P, "orbit"))
        emit(encode_lines(fixed, W, H, P, dev))
        emit(loop_lines(pc, cams, W, H, P, args.loop_frames, dev))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
