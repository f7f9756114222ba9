"""Device time of the four per-frame FLAME kernels (gaussianavatars_b200.flame) at full size, from torch.profiler, with
the bytes each must move and the achieved rate against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  Assets:
synthetic.flame_like_assets (V = 5000 on head_mesh, n_shape = 300, n_expr = 100), 16 timesteps.  One JSON line, with
the GPU it ran on and its power limit.  Run it on its own: tracing slows the host.

    python scripts/flame_kernels.py            (ITERS=500 forward + backward calls)
"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch
from torch.profiler import ProfilerActivity, profile
import gaussianavatars_b200 as g
from gaussianavatars_b200 import synthetic as syn

dev = torch.device("cuda:0")
K = int(os.environ.get("ITERS", 500))
HBM = 3.35e12
a = syn.flame_like_assets(0)
V, NE, T = a["v_template"].shape[0], a["n_expr"], 16
fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=V).items() if k != "dynamic_offset"}
for k in ("expr", "rotation", "neck_pose", "jaw_pose", "eyes_pose", "translation"):
    fp[k].requires_grad_(True)
lbs = g.FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], a["parents"],
                             a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
t_dev = torch.zeros(1, dtype=torch.int32, device=dev)
gv = torch.randn(1, V, 3, device=dev)


def one(i):
    t_dev.fill_(i % T)
    verts, cano = g.flame_pose(lbs, fp, t_dev)
    verts.backward(gv)


for i in range(20):
    one(i)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(K):
        one(i)
    torch.cuda.synchronize()

n3, NB = 3 * V, (V + 31) // 32
pstride = (99 + NE + 3) // 4 * 4
bytes_of = {   # what each kernel must read and write (float32), from the shapes
    "flame_joints_kernel": 4 * (15 * NE + 15 + NE + 18 + 111),
    "flame_skin_kernel": 4 * (NE * n3 + 36 * n3 + 5 * V + n3 + NE + 96 + 2 * n3),
    "flame_skin_backward_kernel": 4 * (NE * n3 + 36 * n3 + 5 * V + n3 + NE + 96 + n3 + NB * pstride + T * (NE + 18)),
    "flame_joints_backward_kernel": 4 * (NB * pstride + 15 * NE + 15 + NE + 18 + NE + 18),
}
times = {k: [0.0, 0] for k in bytes_of}   # total us, launches
for ev in prof.key_averages():
    name = ev.key.split("(")[0]
    for k in bytes_of:
        if name.endswith(k):
            tot = getattr(ev, "device_time_total", None)
            times[k][0] += tot if tot is not None else ev.cuda_time_total
            times[k][1] += ev.count
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip().split("\n")[0]
res = {"what": "flame_kernels", "V": V, "n_expr": NE, "T": T, "calls": K, "gpu": torch.cuda.get_device_name(dev),
       "power_limit": q.split(",")[-1].strip() if q else "unknown"}
for k, (tot, n) in times.items():
    us = tot / max(n, 1)
    res[k] = {"launches": n, "us": round(us, 3), "bytes": bytes_of[k],
              "GBps": round(bytes_of[k] / (us * 1e-6) / 1e9, 1) if us > 0 else None,
              "of_hbm_peak": round(bytes_of[k] / (us * 1e-6) / HBM, 3) if us > 0 else None}
print(json.dumps(res), flush=True)
