"""Cost of drawing the tracked mesh over the avatar (csrc/mesh.cu) -> one JSON line per (setting, arm) on stdout
(appended to profiles/h100/mesh_overlay.jsonl):

  graph_u8        GraphedRender(outputs="u8"): pose, splat forward, display bytes -- one replay per frame
  graph_u8_mesh   GraphedRender(outputs="u8", mesh_opacity=0.5): pose, splat forward (float image), mesh overlay
  fused_overlay   eager mesh_overlay(verts, faces, cam, image) over a prepared float render
  shim_reference  the reference mesh renderer's call order (use_opengl path) on the nvdiffrast shim + render.py's
                  composite in torch, over the same prepared render

Protocol (fps_benchmark_demo.py's): 3 passes of 100 frames after a warm-up pass, CUDA events around each pass, the
median pass reported per frame.  Settings: 100k splats bound to a synthetic FLAME-like head of 9,996 faces, orbit
cameras at 550x802, 1920x1080 and 3840x2160, and a close-up at 550x802 whose nearest faces cover ~1e5 pixels.  The
three mesh kernels' device times come from a separate torch.profiler run over 100 eager overlays.  Every line
carries the card, its power limit and its SM clock, read in the same run."""
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

from gaussianavatars_b200 import mesh_overlay, synthetic as syn  # noqa: E402
from gaussianavatars_b200.flame import FlameLBS  # noqa: E402
from gaussianavatars_b200.graph import GraphedRender  # noqa: E402
from gaussianavatars_b200.model import MeshBoundGaussians  # noqa: E402
from gaussianavatars_b200.renderer import render_display  # noqa: E402
from tests.test_gpu_mesh import _reference_call_order  # noqa: E402

dev = torch.device("cuda:0")
FRAMES, PASSES = 100, 3


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip().split(", ")
    if len(q) != 4:
        return {"gpu": torch.cuda.get_device_name(dev)}
    return {"gpu": q[0], "power_limit_W": float(q[1]), "sm_clock_MHz": float(q[2]), "sm_clock_max_MHz": float(q[3])}


def model(P=100_000, T=8):
    a = syn.flame_like_assets(0)
    fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0]).items()
          if k != "dynamic_offset"}
    lbs = FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                               a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    return MeshBoundGaussians(params, 3, None, None, device=dev, flame=lbs, flame_param=fp)


def cameras(W, H, r, n=8):
    return [syn.orbit_camera(W, H, r=r, fovy_deg=20.0, azimuth_deg=-40 + 80 * i / (n - 1) + (90 if r < 0.5 else 0),
                             elevation_deg=5 * math.sin(i)).to(dev) for i in range(n)]


def timed(step):
    for i in range(FRAMES):   # warm-up pass
        step(i)
    torch.cuda.synchronize()
    ms = []
    for _ in range(PASSES):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(FRAMES):
            step(i)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / FRAMES)
    return sorted(ms)


def main():
    info = gpu_info()
    pc = model()
    bg = torch.ones(3, device=dev)
    F = pc.faces.shape[0]
    for name, W, H, r in (("550x802", 550, 802, 1.0), ("1080p", 1920, 1080, 0.6), ("4k", 3840, 2160, 0.6),
                          ("closeup_550x802", 550, 802, 0.2)):
        cams = cameras(W, H, r)
        lines = []
        for arm, kw in (("graph_u8", {}), ("graph_u8_mesh", {"mesh_opacity": 0.5})):
            view = GraphedRender(pc, W, H, bg, outputs="u8", warm_cameras=cams, warm_timesteps=range(8), **kw)

            def step(i, view=view):
                view.set_inputs(camera=cams[i % len(cams)], timestep=i % 8)
                view.run()

            ms = timed(step)
            assert not view.overflowed() and view.captures == 1
            lines.append({"arm": arm, "ms_per_frame_median": round(ms[1], 4), "ms_per_frame_best": round(ms[0], 4)})
            del view
        # the overlay alone, eager: fused kernels vs the reference's code on the shim, over prepared renders
        renders, verts = [], []
        with torch.no_grad():
            for i, c in enumerate(cams):
                pc.select_mesh_by_timestep(i % 8)
                renders.append(render_display(c, pc, Pipe, bg, 1.0, float_image=True)["render"].clone())
                verts.append(pc.verts.detach().reshape(1, -1, 3).clone())
        faces = pc.faces

        def fused(i):
            k = i % len(cams)
            mesh_overlay(verts[k], faces, cams[k], renders[k])

        def shim(i):
            k = i % len(cams)
            _, _, _, rgba = _reference_call_order(cams[k], verts[k], faces)
            rgba_mesh = rgba.squeeze(0).permute(2, 0, 1)
            out = rgba_mesh[:3] * rgba_mesh[3:] * 0.5 + renders[k] * (rgba_mesh[3:] * (1 - 0.5) + (1 - rgba_mesh[3:]))
            out.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)

        for arm, fn in (("fused_overlay", fused), ("shim_reference", shim)):
            ms = timed(fn)
            lines.append({"arm": arm, "ms_per_frame_median": round(ms[1], 4), "ms_per_frame_best": round(ms[0], 4)})
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(FRAMES):
                fused(i)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            for k in ("mesh_setup_kernel", "mesh_raster_kernel", "mesh_resolve_kernel", "DeviceScan"):
                if k in e.key:
                    kern[k] = round(kern.get(k, 0.0) + e.device_time_total / FRAMES, 2)
        covered = []
        with torch.no_grad():
            for k in range(len(cams)):
                a = mesh_overlay(verts[k], faces, cams[k], torch.zeros(3, H, W, device=dev), mesh_opacity=1.0,
                                 background=(0, 0, 0), out="float")
                covered.append(int((a.abs().sum(0) > 0).sum()))
        # algorithmic bytes of one overlay: faces + vertices read, the u64 winner map written and read (with its
        # memset), the float base read and the u8 frame written
        alg = F * 12 + verts[0].numel() * 4 + W * H * (8 * 3 + 12 + 3)
        for line in lines:
            line.update({"setting": name, "splats": pc._xyz.shape[0], "faces": F, "W": W, "H": H,
                         "frames_per_pass": FRAMES, "passes": PASSES, "mesh_kernel_us": kern,
                         "overlay_algorithmic_bytes": alg, "mean_lit_px": int(sum(covered) / len(covered)), **info})
            print(json.dumps(line), flush=True)
        del renders, verts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
