"""H.264 videos on the device (gaussianavatars_b200.video): one JSON line per measurement to stdout and to --out
(profiles/h100/video.jsonl).

  gpu       the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  encode    gab200_h264_encode on display frames of the synthetic avatar (550x802 with 89k splats, 1920x1080 with
            100k), K = 1, 4, 16, 64 frames per launch and qp 14, 20, 26, 32: CUDA events around enough launches for
            256 frames after warm-up, ms per frame, eager and as a replayed CUDA graph; mean sample bytes; Y-PSNR of
            FFmpeg's decode of the file (the encoder's reconstruction, bit for bit) against the source's Y plane
  kernels   each kernel's share of one encode at qp 20, K = 1 and 16 (torch.profiler, a run of its own): the
            per-diagonal h264_mb_kernel launches against the rest
  loop      render.py's loop: a GraphedRender replay per frame into a VideoWriter, the file on disk; the same frames
            as device PNG files (GraphedRender(png=True), host_png); frames per second
  mp4v      OpenCV's MPEG-4 Part 2 writer on the same frames (host copies included) -- a different codec, for
            orientation only

    python scripts/video_sweep.py --out profiles/h100/video.jsonl
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

from png_sweep import avatar, displays, gpu_info, loop_lines  # noqa: E402

SIZES = ((550, 802, 89_000), (1920, 1080, 100_000))
KS = (1, 4, 16, 64)
QPS = (14, 20, 26, 32)


def source_y(frames: np.ndarray) -> np.ndarray:
    """BT.601 limited-range Y of (K,H,W,3) uint8, the encoder's formula."""
    r, g, b = (frames[..., c].astype(np.int64) for c in range(3))
    return ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16


def decoded_y(data: bytes, H: int, W: int) -> list:
    import cv2
    with tempfile.NamedTemporaryFile(suffix=".mp4") as f:
        f.write(data)
        f.flush()
        cap = cv2.VideoCapture(f.name)
        cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
        out = []
        while True:
            ok, y = cap.read()
            if not ok:
                break
            out.append(y.reshape(H, W))
    return out


def time_encode(frames, qp, dev, graph: bool, total_frames=256):
    from gaussianavatars_b200 import video as V
    K, H, W = V.check_frames(frames)
    sc = V.scratch(K, H, W, dev)
    out = torch.empty((K, V.slot_stride(W, H)), dtype=torch.uint8, device=dev)
    lens = torch.empty(K, dtype=torch.int64, device=dev)
    n = max(4, total_frames // K)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            V.launch_encode(frames, qp, sc, out, lens)
        g = None
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                V.launch_encode(frames, qp, sc, out, lens)
            g.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(n):
            if g is not None:
                g.replay()
            else:
                V.launch_encode(frames, qp, sc, out, lens)
        b.record(s)
        torch.cuda.synchronize()
    return a.elapsed_time(b) / n / K, float(lens.double().mean())


def encode_lines(frames64, W, H, P, dev):
    from gaussianavatars_b200 import encode_video
    out = []
    src_y = source_y(frames64[:4].cpu().numpy())
    for qp in QPS:
        ys = decoded_y(encode_video(frames64[:4], qp=qp), H, W)
        mse = np.mean([(y.astype(np.float64) - s) ** 2 for y, s in zip(ys, src_y)])
        psnr = float(10 * np.log10(255.0 ** 2 / mse)) if mse > 0 else float("inf")
        for K in KS:
            fr = frames64[:K].contiguous()
            ms, mean_bytes = time_encode(fr, qp, dev, graph=False)
            ms_g, _ = time_encode(fr, qp, dev, graph=True)
            out.append({"kind": "encode", "width": W, "height": H, "splats": P, "frames_per_launch": K, "qp": qp,
                        "ms_per_frame": ms, "ms_per_frame_graph": ms_g, "mean_sample_bytes": mean_bytes,
                        "raw_rgb_bytes": W * H * 3, "y_psnr_db": psnr, "psnr_frames": len(ys)})
    return out


def kernel_lines(frames64, W, H, dev):
    from torch.profiler import ProfilerActivity, profile
    from gaussianavatars_b200 import video as V
    out = []
    for K in (1, 16):
        fr = frames64[:K].contiguous()
        sc = V.scratch(K, H, W, dev)
        buf = torch.empty((K, V.slot_stride(W, H)), dtype=torch.uint8, device=dev)
        lens = torch.empty(K, dtype=torch.int64, device=dev)
        V.launch_encode(fr, 20, sc, buf, lens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                V.launch_encode(fr, 20, sc, buf, lens)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            if "h264_" in e.key:
                name = "h264_" + e.key.split("h264_", 1)[1].split("(")[0].split("E")[0]
                t = getattr(e, "device_time_total", None)
                t = e.cuda_time_total if t is None else t
                per[name] = per.get(name, 0.0) + t / 1e3 / 10
        total = sum(per.values())
        out.append({"kind": "kernels", "width": W, "height": H, "frames_per_launch": K, "qp": 20,
                    "ms_per_launch": per, "diagonal_share": per.get("h264_mb_kernel", 0.0) / total if total else None,
                    "diagonal_launches": (W + 15) // 16 + (H + 15) // 16 - 1})
    return out


def video_loop(pc, cams, W, H, P, frames_n, dev):
    from gaussianavatars_b200 import VideoWriter
    from gaussianavatars_b200.graph import GraphedRender
    view = GraphedRender(pc, W, H, torch.ones(3), outputs="u8", warm_cameras=cams)
    for i in range(4):
        view.set_inputs(camera=cams[i % 16])
        view.run(check=True)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "renders.mp4")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with VideoWriter(path, W, H, fps=25, qp=20, batch=16) as vw:
            for i in range(frames_n):
                view.set_inputs(camera=cams[i % 16])
                view.run()
                vw.add(view.display)
        sec = time.perf_counter() - t0
        size = os.path.getsize(path)
        import cv2
        cap = cv2.VideoCapture(path)
        opened = [int(cap.get(cv2.CAP_PROP_FRAME_COUNT)), cap.get(cv2.CAP_PROP_FPS),
                  int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))]
    return {"kind": "loop", "mode": "video", "width": W, "height": H, "splats": P, "frames": frames_n, "qp": 20,
            "batch": 16, "frames_per_s": frames_n / sec, "file_bytes": size,
            "ffmpeg_opens_as": dict(zip(("frames", "fps", "width", "height"), opened))}


def mp4v_line(frames64, W, H, P):
    import cv2
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "mp4v.mp4")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 25, (W, H))
        if not vw.isOpened():
            return {"kind": "mp4v", "width": W, "height": H, "opened": False}
        for f in frames64:
            vw.write(np.ascontiguousarray(f.cpu().numpy()[..., ::-1]))
        vw.release()
        sec = time.perf_counter() - t0
        size = os.path.getsize(path)
    return {"kind": "mp4v", "codec": "MPEG-4 Part 2 (OpenCV mp4v, CPU)", "width": W, "height": H, "splats": P,
            "frames": len(frames64), "frames_per_s": len(frames64) / sec, "file_bytes": size}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--loop-frames", type=int, default=64)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the sweep measures on a GPU"
    dev = torch.device("cuda:0")
    lines = [gpu_info()]
    for W, H, P in SIZES:
        pc, cams = avatar(P, W, H, dev)
        frames64 = displays(pc, cams, dev).repeat(4, 1, 1, 1).contiguous()
        lines += encode_lines(frames64, W, H, P, dev)
        lines += kernel_lines(frames64, W, H, dev)
        lines.append(video_loop(pc, cams, W, H, P, args.loop_frames, dev))
        lines += [ln for ln in loop_lines(pc, cams, W, H, P, args.loop_frames, dev) if ln["mode"] == "png"]
        lines.append(mp4v_line(frames64, W, H, P))
        for ln in lines[-8:]:
            print(json.dumps(ln), flush=True)
    sink = open(args.out, "w") if args.out else None
    for line in lines:
        if sink:
            sink.write(json.dumps(line) + "\n")
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
