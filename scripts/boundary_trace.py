"""Kernel boundaries of the headline step: every kernel, memset and memcpy node of one graph replay, in order, with the
idle gap in front of each.

    python scripts/boundary_trace.py [--replays 50] [--out profiles/h100/boundaries.jsonl] [--arm NAME]

The step is bench.py's: 100k bound splats, 1920x1080, SH degree 3, face frame + fused forward + backward down to the
raw parameters and the mesh vertices, one GraphedFrame replay, the L2 flushed between replays.  torch.profiler (CUDA
activities) records the replays; the nodes of replay r are the GPU activities whose correlation id is that replay's
cudaGraphLaunch.  Per node the output gives the median over replays of its start (from the replay's first node), its
duration and the gap from the end of the previous node to its start (negative: the two overlap, as with programmatic
dependent launch).  Lines appended to --out: a header (card, power limit, clocks, read in this same process), one line
per node, one summary (sum of positive gaps, sum of node durations, replay span: first start to last end).  The
profiler perturbs the host, not the order or the count of the nodes; take step times from bench.py.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    """Name, power limit (W) and SM clocks of cuda:0, read with nvidia-smi's query interface."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_mhz": int(out[2]), "sm_max_mhz": int(out[3])}
    except Exception as e:  # no nvidia-smi: the name at least
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "card_query_error": str(e)}


def build_frame(dev):
    import bench as B
    from gaussianavatars_b200 import rasterizer as R
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.graph import GraphedFrame, camera_block
    from gaussianavatars_b200.model import MeshBoundGaussians

    R.keep_last_state(False)
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(B.P_SPLATS, n_faces=faces.shape[0], seed=0, sh_degree=B.SH_DEGREE)
    pc = MeshBoundGaussians(params, B.SH_DEGREE, verts, faces, pose_fn=syn.pose_mesh, device=dev, requires_grad=True)
    cams = [c.to(dev) for c in B.make_cameras(B.N_CAMERAS)]
    posed = [syn.pose_mesh(pc.verts_rest, c.timestep).contiguous() for c in cams]
    blocks = [camera_block(c) for c in cams]
    bg = torch.ones(3, device=dev)
    gout = torch.randn(3, B.HEIGHT, B.WIDTH, generator=torch.Generator().manual_seed(1)).to(dev) / (3 * B.HEIGHT * B.WIDTH)
    c0 = cams[0]
    fr = GraphedFrame(pc, B.WIDTH, B.HEIGHT, c0.FoVx, c0.FoVy, bg, loss="dL_dimage", warm_cameras=blocks)
    fr.set_inputs(camera=blocks[0], verts=posed[0], dL_dimage=gout)
    fr.capture()

    def step(i):
        fr.set_inputs(camera=blocks[i % len(blocks)], verts=posed[i % len(posed)])
        fr.run()

    return fr, step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "boundaries.jsonl"))
    ap.add_argument("--arm", default="", help="label written into every line (e.g. the commit measured)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "boundary_trace.py needs a GPU"
    dev = torch.device("cuda", 0)
    from gaussianavatars_b200 import _native as N

    N.lib()
    fr, step = build_frame(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for i in range(10):
        flush.fill_(i & 0xFF)
        step(i)
    torch.cuda.synchronize(dev)

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(a.replays):
            flush.fill_(i & 0xFF)
            step(i)
        torch.cuda.synchronize(dev)
    assert not fr.overflowed(wait=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]

    launches = {e["args"]["correlation"] for e in events
                if e.get("ph") == "X" and e.get("name") == "cudaGraphLaunch" and "correlation" in e.get("args", {})}
    kinds = {"kernel": "kernel", "gpu_memset": "memset", "gpu_memcpy": "memcpy"}
    replays = {}
    for e in events:
        if e.get("ph") == "X" and e.get("cat") in kinds and e.get("args", {}).get("correlation") in launches:
            replays.setdefault(e["args"]["correlation"], []).append(
                (float(e["ts"]), float(e["dur"]), kinds[e["cat"]], e["name"], e["args"].get("stream")))
    seqs = [sorted(v) for _, v in sorted(replays.items())]
    n_nodes = statistics.mode(len(s) for s in seqs)
    seqs = [s for s in seqs if len(s) == n_nodes]
    assert seqs, "no graph replay was traced"

    head = {"kind": "header", "arm": a.arm, **card(), "torch": torch.__version__, "replays_traced": len(seqs),
            "nodes_per_replay": n_nodes, "step": "bench.py headline step: one GraphedFrame replay, L2 flushed between "
            "replays", "command": "python scripts/boundary_trace.py " + " ".join(sys.argv[1:])}
    lines = [head]
    gap_sums, dur_sums, spans, med_gaps = [], [], [], []
    for k in range(n_nodes):
        starts = [s[k][0] - s[0][0] for s in seqs]
        durs = [s[k][1] for s in seqs]
        gaps = [s[k][0] - (s[k - 1][0] + s[k - 1][1]) for s in seqs] if k else [0.0] * len(seqs)
        med_gaps.append(statistics.median(gaps))
        ts, du, kind, name, stream = seqs[0][k]
        lines.append({"kind": kind, "arm": a.arm, "index": k, "name": name[:160], "stream": stream,
                      "start_us": round(statistics.median(starts), 2), "dur_us": round(statistics.median(durs), 2),
                      "gap_before_us": round(med_gaps[-1], 2)})
    for s in seqs:
        gap_sums.append(sum(max(0.0, s[k][0] - (s[k - 1][0] + s[k - 1][1])) for k in range(1, len(s))))
        dur_sums.append(sum(x[1] for x in s))
        spans.append(max(x[0] + x[1] for x in s) - s[0][0])
    counts = {}
    for ln in lines[1:]:
        counts[ln["kind"]] = counts.get(ln["kind"], 0) + 1
    lines.append({"kind": "summary", "arm": a.arm, "nodes": counts,
                  "gap_sum_us_median": round(statistics.median(gap_sums), 2),
                  "gap_sum_us_min_max": [round(min(gap_sums), 2), round(max(gap_sums), 2)],
                  "node_dur_sum_us_median": round(statistics.median(dur_sums), 2),
                  "memset_memcpy_dur_us": round(sum(ln["dur_us"] for ln in lines[1:] if ln["kind"] != "kernel"), 2),
                  "span_us_median": round(statistics.median(spans), 2),
                  "note": "gap = start of a node - end of the node before it (profiled replays; negative = overlap)"})
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "a") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")
    for ln in lines:
        if ln["kind"] in ("header", "summary"):
            print(json.dumps(ln))
        else:
            print(f'{ln["index"]:3d} {ln["kind"]:7s} start {ln["start_us"]:8.2f} dur {ln["dur_us"]:7.2f} '
                  f'gap {ln["gap_before_us"]:6.2f}  {ln["name"][:90]}')


if __name__ == "__main__":
    main()
