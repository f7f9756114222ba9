"""I_NxN macroblocks in the device H.264 encoder (VideoWriter(intra4x4=True), gab200_h264_encode_flags), off against
on: one JSON line per measurement to stdout and to --out (profiles/h100/video_intra4x4.jsonl).

  gpu     the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  size    bytes per frame, Y-PSNR of FFmpeg's decode against the source's Y plane and the share of macroblocks coded
          I_NxN, intra4x4 off and on, qp 20, 26, 32, 38, gop 1 and 25, deblock off and on, on 64 display frames of the
          synthetic avatar (550x802 with 89k splats, 1920x1080 with 100k) whose timestep advances under a fixed camera
          ("fixed") and under an orbiting one ("orbit")
  encode  ms per frame at gop 25 and qp 26, K = 1, 16, 64 frames per launch, eager and as a replayed CUDA graph,
          intra4x4 off and on alternated in the same run (CUDA events around enough launches for 256 frames)
  loop    render.py's loop with gop 25 and qp 26, intra4x4 off and on: a GraphedRender replay per frame (fixed camera,
          timestep advancing) into a VideoWriter, the file on disk; frames per second
  bias    (--bias, no GPU) the I4_BIAS candidates: tests/h264_intra4x4_oracle.py, which equals the device bit for
          bit, run with each candidate on one IDR frame of tests/h264_corpus.avatar_like at 550x802: bytes, Y-PSNR of
          the reconstruction and the I_NxN share ("bias": null is I_16x16 alone)

    python scripts/video_intra4x4_sweep.py --out profiles/h100/video_intra4x4.jsonl
    python scripts/video_intra4x4_sweep.py --bias --out bias.jsonl
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

SIZES = ((550, 802, 89_000), (1920, 1080, 100_000))
KS = (1, 16, 64)
QPS = (20, 26, 32, 38)
GOP = 25
BIASES = (None, -8, 0, 8, 16)


def info_offset(H: int, W: int) -> int:
    """The byte offset of the macroblocks' info words in a frame's scratch (csrc/h264.cu layout(): the source and
    reconstructed planes, the TotalCoeff and the levels come before it, each 256-byte aligned)."""
    def al(x):
        return (x + 255) // 256 * 256
    nmb = ((W + 15) // 16) * ((H + 15) // 16)
    o = al(384 * nmb)
    o = al(o + 384 * nmb)
    o = al(o + 24 * nmb)
    return al(o + 27 * 32 * nmb)


def i4_share(frames, qp, gop, deblock, dev) -> float:
    """The share of the clip's macroblocks coded I_NxN (info bit 14), read back from the scratch."""
    import torch
    from gaussianavatars_b200 import video as V
    K, H, W = V.check_frames(frames)
    sc = V.flags_scratch(K, H, W, gop, deblock, True, dev)
    out = torch.empty((K, V.slot_stride(W, H, gop)), dtype=torch.uint8, device=dev)
    lens = torch.empty(K, dtype=torch.int64, device=dev)
    V.launch_encode_flags(frames, qp, gop, deblock, True, V.state_buffer(H, W, dev), sc, out, lens)
    nmb = ((W + 15) // 16) * ((H + 15) // 16)
    stride, off = sc.numel() // K, info_offset(H, W)
    info = sc.view(K, stride)[:, off:off + 4 * nmb].contiguous().view(torch.int32).cpu().numpy()
    assert (info >> 15 == 0).all()
    return float(((info >> 14) & 1).mean())


def size_lines(frames, W, H, P, motion, dev):
    from gaussianavatars_b200 import encode_video
    from video_sweep import decoded_y, source_y
    src = source_y(frames.cpu().numpy())
    out = []
    for qp in QPS:
        for gop in (1, GOP):
            for deblock in (False, True):
                for intra4x4 in (False, True):
                    data = encode_video(frames, qp=qp, gop=gop, deblock=deblock, intra4x4=intra4x4)
                    ys = decoded_y(data, H, W)
                    mse = np.mean([(y.astype(np.float64) - s) ** 2 for y, s in zip(ys, src)])
                    out.append({"kind": "size", "width": W, "height": H, "splats": P, "motion": motion, "qp": qp,
                                "gop": gop, "deblock": deblock, "intra4x4": intra4x4, "frames": len(frames),
                                "decoded_frames": len(ys), "bytes_per_frame": len(data) / len(frames),
                                "y_psnr_db": float(10 * np.log10(255 ** 2 / mse)) if mse else None,
                                "i4_share": i4_share(frames, qp, gop, deblock, dev) if intra4x4 else 0.0})
    return out


def time_stream(frames, qp, gop, intra4x4, dev, graph, total_frames=256):
    import torch
    from gaussianavatars_b200 import video as V
    K, H, W = V.check_frames(frames)
    st = V.state_buffer(H, W, dev)
    sc = V.flags_scratch(K, H, W, gop, False, intra4x4, dev)
    out = torch.empty((K, V.slot_stride(W, H, gop)), dtype=torch.uint8, device=dev)
    lens = torch.empty(K, dtype=torch.int64, device=dev)

    def launch():
        V.launch_encode_flags(frames, qp, gop, False, intra4x4, st, sc, out, lens)

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
            for intra4x4 in (False, True, False, True):        # alternated: each mode measured twice
                ms = time_stream(frames64[:K].contiguous(), 26, GOP, intra4x4, dev, graph)
                out.append({"kind": "encode", "width": W, "height": H, "splats": P, "gop": GOP, "qp": 26, "K": K,
                            "graph": graph, "intra4x4": intra4x4, "ms_per_frame": ms})
    return out


def loop_lines(pc, cams, W, H, P, frames_n, dev):
    import torch
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
    for intra4x4 in (False, True, False, True):
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "renders.mp4")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with VideoWriter(path, W, H, fps=25, qp=26, batch=16, gop=GOP, intra4x4=intra4x4) as vw:
                for i in range(frames_n):
                    view.set_inputs(camera=cams[0], verts=poses[i % 8])
                    view.run()
                    vw.add(view.display)
            sec = time.perf_counter() - t0
            size = os.path.getsize(path)
        out.append({"kind": "loop", "mode": "video", "width": W, "height": H, "splats": P, "frames": frames_n,
                    "qp": 26, "batch": 16, "gop": GOP, "intra4x4": intra4x4, "frames_per_s": frames_n / sec,
                    "file_bytes": size})
    return out


def bias_lines():
    from oracle import h264 as O
    from tests import h264_corpus as hc
    from tests import h264_intra4x4_oracle as I
    W, H = 550, 802
    img = hc.avatar_like(W, H)
    src = O.rgb_to_yuv(img)[0][:H, :W].astype(np.float64)
    keep = I.I4_BIAS
    out = []
    try:
        for qp in QPS:
            for bias in BIASES:
                I.I4_BIAS = 1 << 40 if bias is None else bias
                f = I.encode_stream(img[None], qp, 1)[0]
                mse = np.mean((I.crop(f["recon"], W, H)[0].astype(np.float64) - src) ** 2)
                out.append({"kind": "bias", "source": "oracle", "image": "avatar_like", "width": W, "height": H,
                            "qp": qp, "gop": 1, "bias": bias, "bytes_per_frame": len(f["sample"]),
                            "y_psnr_db": float(10 * np.log10(255 ** 2 / mse)),
                            "i4_share": float((f["types"] == "I4").mean())})
    finally:
        I.I4_BIAS = keep
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the lines to this file")
    ap.add_argument("--loop-frames", type=int, default=400)
    ap.add_argument("--bias", action="store_true", help="the I4_BIAS candidates through the oracle (no GPU)")
    ap.add_argument("--width", type=int, default=None, help="only the size of this width")
    args = ap.parse_args()
    lines = []

    def emit(new):
        for ln in new:
            print(json.dumps(ln), flush=True)
        lines.extend(new)

    if args.bias:
        emit(bias_lines())
    else:
        import torch
        from png_sweep import avatar, gpu_info
        from video_gop_sweep import clip
        dev = torch.device("cuda")
        emit([gpu_info()])
        for W, H, P in SIZES:
            if args.width not in (None, W):
                continue
            pc, cams = avatar(P, W, H, dev)
            fixed = clip(pc, cams, dev, orbit=False)
            emit(size_lines(fixed, W, H, P, "fixed", dev))
            emit(size_lines(clip(pc, cams, dev, orbit=True), W, H, P, "orbit", dev))
            emit(encode_lines(fixed, W, H, P, dev))
            emit(loop_lines(pc, cams, W, H, P, args.loop_frames, dev))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
