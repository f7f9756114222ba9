"""The local viewer's trajectory export on the device (trajectory.export_trajectory) against the reference's loop: one
JSON line per measurement to stdout and to --out (profiles/h100/trajectory.jsonl).

  gpu     the card's name, power limit and max SM clock (nvidia-smi, read in the same run)
  export  frames/s of three arms over one 100-frame path (two keyframes, 60 degrees of orbit, the "dynamic" timestep
          advancing over a 16-timestep FLAME sequence), at the viewer's default 960x540 and at 1920x1080, with and
          without the mesh (opacity 0.5), on a 100k-splat synthetic FLAME avatar; every arm writes its PNG files to a
          temporary directory:
            device     export_trajectory(): one scheduled GraphedRender (quantize="viewer", png=True), the files from
                       the pinned ring, one synchronisation per 16 frames; the capture and warm-up included
            reference  the viewer's export loop in one thread: eager render() (the float image), the mesh composited
                       in torch over it, .cpu(), (np.clip(rgb, 0, 1) * 255).astype(np.uint8), PIL save
            eager      render_display(quantize="viewer") per frame (with the mesh: the float image and mesh_overlay's
                       bytes), .cpu(), PIL save
          median of 3 passes after one warm-up pass; wall clock around work that ends in a synchronisation.  The host
          arms, whose PIL encode takes tenths of a second per frame, time the path's first 25 frames per pass.

    python scripts/trajectory_sweep.py --out profiles/h100/trajectory.jsonl
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from png_sweep import Pipe, gpu_info  # noqa: E402

SIZES = ((960, 540), (1920, 1080))
P, T, FRAMES, PASSES, HOST_FRAMES = 100_000, 16, 100, 3, 25


def flame_avatar(dev):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.flame import FlameLBS
    from gaussianavatars_b200.model import MeshBoundGaussians
    a = syn.flame_like_assets(0)
    fp = syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0])
    fp.pop("dynamic_offset")
    lbs = FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                               a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    return MeshBoundGaussians(params, 3, None, None, device=dev, flame=lbs,
                              flame_param={k: v.to(dev).contiguous() for k, v in fp.items()})


def camera_path(W, H):
    from scipy.spatial.transform import Rotation
    from gaussianavatars_b200.trajectory import CameraPath, keyframe
    rot = Rotation.from_euler("y", [[-30.0], [30.0]], degrees=True).as_matrix()
    kfs = [keyframe(rot[0], np.zeros(3, np.float32), 1.0, 20.0, FRAMES), keyframe(rot[1], np.zeros(3, np.float32),
                                                                                 1.0, 20.0, FRAMES)]
    return CameraPath(kfs, width=W, height=H, dynamic=True, num_timesteps=T)


def device_arm(pc, path, bg, mesh, out):
    from gaussianavatars_b200.trajectory import export_trajectory
    export_trajectory(pc, path, out, bg=bg, mesh_opacity=0.5 if mesh else None)


def cams_of(path, dev):
    from types import SimpleNamespace
    out = []
    for i in range(len(path)):
        c = path.camera(i)
        out.append(SimpleNamespace(**{k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in vars(c).items()}))
    return out


@torch.no_grad()
def reference_arm(pc, path, cams, bg, mesh, out):
    from PIL import Image
    from gaussianavatars_b200 import mesh_overlay
    from gaussianavatars_b200.renderer import render
    rows = path.rows().to(bg.device)
    for i, cam in enumerate(cams[:HOST_FRAMES]):
        pc.select_mesh_by_timestep(path.timestep(i))
        rgb = render(cam, pc, Pipe, bg)["render"]
        if mesh:   # the float composite of render.py's / the viewer's expression
            rgb = mesh_overlay(pc.verts, pc.faces, rows[i], rgb, mesh_opacity=0.5, out="float")
        buf = rgb.permute(1, 2, 0).contiguous().cpu().numpy()
        Image.fromarray((np.clip(buf, 0, 1) * 255).astype(np.uint8)).save(os.path.join(out, f"{i:05d}.png"))


@torch.no_grad()
def eager_arm(pc, path, cams, bg, mesh, out):
    from PIL import Image
    from gaussianavatars_b200 import mesh_overlay
    from gaussianavatars_b200.renderer import render_display
    rows = path.rows().to(bg.device)
    for i, cam in enumerate(cams[:HOST_FRAMES]):
        pc.select_mesh_by_timestep(path.timestep(i))
        r = render_display(cam, pc, Pipe, bg, float_image=mesh, quantize="viewer")
        u8 = mesh_overlay(pc.verts, pc.faces, rows[i], r["render"], mesh_opacity=0.5) if mesh else r["display_u8"]
        Image.fromarray(u8.cpu().numpy()).save(os.path.join(out, f"{i:05d}.png"))


def timed(fn):
    runs = []
    for k in range(PASSES + 1):
        with tempfile.TemporaryDirectory() as out:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(out)
            torch.cuda.synchronize()
            runs.append(time.perf_counter() - t0)
    return runs[1:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lines = [gpu_info()]
    print(json.dumps(lines[0]), flush=True)
    sink = open(args.out, "w") if args.out else None
    if sink:
        sink.write(json.dumps(lines[0]) + "\n")
    pc = flame_avatar(dev)
    bg = torch.ones(3, device=dev)
    for W, H in SIZES:
        path = camera_path(W, H)
        cams = cams_of(path, dev)
        for mesh in (False, True):
            arms = {"device": lambda o: device_arm(pc, path, bg, mesh, o),
                    "reference": lambda o: reference_arm(pc, path, cams, bg, mesh, o),
                    "eager": lambda o: eager_arm(pc, path, cams, bg, mesh, o)}
            for name, fn in arms.items():
                runs = timed(fn)
                med = statistics.median(runs)
                n = len(path) if name == "device" else min(HOST_FRAMES, len(path))
                lines.append({"kind": "export", "arm": name, "width": W, "height": H, "mesh": mesh, "splats": P,
                              "frames": n, "passes_s": [round(r, 4) for r in runs],
                              "median_s": round(med, 4), "frames_per_s": round(n / med, 1)})
                print(json.dumps(lines[-1]), flush=True)
                if sink:
                    sink.write(json.dumps(lines[-1]) + "\n")
                    sink.flush()
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
