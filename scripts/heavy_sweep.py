"""Blend heavy/light threshold sweep on the headline workload: blend_fwd / blend_bwd stage times for every pair of a
forward threshold (HEAVY_FWD, GAB200_TUNE_HEAVY_FWD) and a backward threshold (HEAVY_BWD, GAB200_TUNE_HEAVY_BWD).
Both are comma-separated lists; the default HEAVY_BWD is the library's default, so a plain run sweeps the forward only.
The strip masks the backward reads are written by whichever forward schedule ran; a backward threshold changes only the
order in which the gradients are summed, so the largest gradient difference against the first pair is printed too."""
import json, math, os, sys
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch
from gaussianavatars_b200 import synthetic as syn, _native as N
from gaussianavatars_b200.model import MeshBoundGaussians
from gaussianavatars_b200.renderer import render

dev = torch.device("cuda:0")
class Pipe: debug = False; compute_cov3D_python = False; convert_SHs_python = False
P, W, H = int(os.environ.get("P", 100000)), int(os.environ.get("W", 1920)), int(os.environ.get("H", 1080))
verts, faces = syn.head_mesh()
params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=0, sh_degree=3)
pc = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=dev, requires_grad=True)
cams = [syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=-60 + 120 * (i + .5) / 16, elevation_deg=5 * math.sin(i)).to(dev) for i in range(16)]
posed = [syn.pose_mesh(pc.verts_rest, i).contiguous().requires_grad_(True) for i in range(16)]
bg = torch.ones(3, device=dev)
gout = torch.randn(3, H, W, generator=torch.Generator().manual_seed(1)).to(dev) / (3 * H * W)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

def step(i):
    for p in pc.parameters(): p.grad = None
    pc.update_mesh_properties(posed[i % 16])
    out = render(cams[i % 16], pc, Pipe, bg)
    out["render"].backward(gout)
    return out

def knob_values(name, default):
    return [int(x) for x in os.environ.get(name, default).split(",")]

ref = ref_g = None
for hf in knob_values("HEAVY_FWD", "32,96,192,384,768,100000"):
    for hb in knob_values("HEAVY_BWD", "2048"):
        N.tune(N.TUNE_HEAVY_FWD, hf); N.tune(N.TUNE_HEAVY_BWD, hb)
        for i in range(6): step(i)
        img = step(0)["render"].detach().clone()
        g = torch.cat([p.grad.reshape(-1) for p in pc.parameters()]).clone()
        if ref is None: ref, ref_g = img, g
        same = bool(torch.equal(ref, img))
        diff = float((g - ref_g).abs().max() / ref_g.abs().max())
        N.stage_timing(True); N.stage_times(True)
        for i in range(40):
            flush.fill_(i & 255); step(i); torch.cuda.synchronize()
        st = N.stage_times(True); N.stage_timing(False)
        print(json.dumps({"heavy_fwd": hf, "heavy_bwd": hb,
                          "blend_fwd_us": round(st["blend_fwd"][0] / st["blend_fwd"][1] * 1e3, 1),
                          "blend_bwd_us": round(st["blend_bwd"][0] / st["blend_bwd"][1] * 1e3, 1),
                          "image_identical": same, "max_grad_diff_vs_first": diff}), flush=True)
