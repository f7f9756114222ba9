"""BASELINE.json config 5: the fps_benchmark_demo.py protocol (3 rounds x n_iter, forward only under no_grad, CUDA
events; reference: fps_benchmark_demo.py:53-66) over 50k/100k/300k/1M splats x 720p/1080p/4K, with and without the
per-frame mesh-frame update inside the timed region.  One JSON line per cell -> profiles/<round>/fps_sweep.jsonl.

Arms (same cells, same protocol):
  eager          render() under no_grad, one eager call per frame (the reference's loop)
  graph          GraphedRender(outputs="float"): one forward-only graph replay per frame, float (3,H,W) image
  graph_u8       GraphedRender(outputs="u8"): the blend writes the display (H,W,3) uint8 image only
  graph_u8_host  graph_u8 + the frame on the host through a 2-slot pinned ring, the consumer one replay behind
With the mesh update in the loop the graph arms run update_mesh_properties inside the replay.
A last line ("demo") is fps_benchmark_demo.py's own setting: 550x802, fovy 20 deg, radius 1, white background, a
FLAME head (synthetic.flame_like_assets) with the timestep advancing every frame and the pose inside the replay.
Every line carries the GPU, its power limit and SM clocks (sampled right after the cell) and how many runs it had."""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch
from gaussianavatars_b200 import synthetic as syn, rasterizer as R
from gaussianavatars_b200.graph import GraphedRender
from gaussianavatars_b200.model import MeshBoundGaussians
from gaussianavatars_b200.renderer import render

dev = torch.device("cuda:0")
class Pipe: debug=False; compute_cov3D_python=False; convert_SHs_python=False
peak = 6585.8
try: peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception: pass
sizes = [int(x) for x in os.environ.get("SWEEP_P", "50000,100000,300000,1000000").split(",")]
res = {"720p": (1280, 720), "1080p": (1920, 1080), "4K": (3840, 2160)}
n_iter = int(os.environ.get("SWEEP_ITERS", "100"))
arms = os.environ.get("SWEEP_ARMS", "eager,graph,graph_u8,graph_u8_host").split(",")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_W": float(q[1]), "sm_clock_MHz": int(q[2]), "sm_clock_max_MHz": int(q[3])} \
        if len(q) == 4 else {"gpu": torch.cuda.get_device_name(dev)}


def graph_rounds(view, n_iter, host, step=None):
    """3 rounds of n_iter replays: frames per second of each round."""
    fps = []
    for rnd in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n_iter):
            if step is not None: step(i)
            view.run()
            if host and i > 0: view.host_frame(view.replays - 2)   # the consumer reads the previous frame
        if host: view.host_frame()
        e1.record(); torch.cuda.synchronize()
        fps.append(n_iter / (e0.elapsed_time(e1) / 1e3))
    assert not view.overflowed(), "a timed replay overflowed its capacity"
    return sorted(fps)


verts, faces = syn.head_mesh()
bg = torch.ones(3, device=dev)
R.keep_last_state(True)
for P in sizes:
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, verts, faces, device=dev)
    pc.select_mesh_by_timestep(0)
    for name, (W, H) in res.items():
        cam = syn.orbit_camera(W, H).to(dev)
        with torch.no_grad():
            for _ in range(5): render(cam, pc, Pipe, bg)
            _, _, _, n = R.export_last_binning()
        for arm in arms:
            for with_mesh in (False, True):
                if arm == "eager":
                    fps = []
                    with torch.no_grad():
                        for rnd in range(3):
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            for _ in range(n_iter):
                                if with_mesh: pc.update_mesh_properties(pc.verts)
                                render(cam, pc, Pipe, bg)["render"]
                            e1.record(); torch.cuda.synchronize()
                            fps.append(n_iter / (e0.elapsed_time(e1) / 1e3))
                    fps.sort()
                    out_bytes = H * W * 12
                else:
                    host = arm == "graph_u8_host"
                    view = GraphedRender(pc, W, H, bg, outputs="float" if arm == "graph" else "u8",
                                         mesh_update=with_mesh, host_slots=2 if host else 0, warm_cameras=[cam])
                    view.set_inputs(camera=cam, verts=pc.verts)
                    for _ in range(5): view.run(check=True)
                    fps = graph_rounds(view, n_iter, host)
                    out_bytes = H * W * (12 if arm == "graph" else 3)
                    del view
                    pc.select_mesh_by_timestep(0)
                alg = P * 240 + P * 48 + n * 12 + n * 24 + n * 40 + out_bytes  # SURVEY 8(d) forward (inference) bytes
                gbs = alg * fps[1] / 1e9
                print(json.dumps({"arm": arm, "splats": P, "res": name, "W": W, "H": H, "instances": int(n),
                                  "mesh_update_in_loop": with_mesh, "fps_median": round(fps[1], 1),
                                  "fps_best": round(fps[2], 1), "ms_median": round(1e3 / fps[1], 4),
                                  "algorithmic_GBps": round(gbs, 1), "frac_of_measured_hbm_peak": round(gbs / peak, 4),
                                  "rounds": 3, "iters_per_round": n_iter, "runs": 1, **gpu_info()}), flush=True)
    del pc
    torch.cuda.empty_cache()

# ---- fps_benchmark_demo.py's setting with a FLAME head: the timestep advances every frame -----------------------------
if os.environ.get("SWEEP_DEMO", "1") == "1":
    from gaussianavatars_b200.flame import FlameLBS
    T, P_demo, W, H = 64, 89_021, 550, 802
    n_demo = int(os.environ.get("SWEEP_DEMO_ITERS", "500"))
    a = syn.flame_like_assets(0)
    fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0]).items()
          if k != "dynamic_offset"}
    lbs = FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                               a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
    params = syn.avatar_splats(P_demo, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, None, None, device=dev, flame=lbs, flame_param=fp)
    cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0).to(dev)
    lines = []
    for arm in ("eager", "graph_u8"):
        if arm == "eager":
            fps = []
            with torch.no_grad():
                for t in range(5): pc.select_mesh_by_timestep(t % T); render(cam, pc, Pipe, bg)
                for rnd in range(3):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for i in range(n_demo):
                        pc.select_mesh_by_timestep(i % T)
                        render(cam, pc, Pipe, bg)["render"]
                    e1.record(); torch.cuda.synchronize()
                    fps.append(n_demo / (e0.elapsed_time(e1) / 1e3))
            fps.sort()
        else:
            view = GraphedRender(pc, W, H, bg, outputs="u8", warm_cameras=[cam])
            view.set_inputs(camera=cam, timestep=0)
            for t in range(5): view.set_inputs(timestep=t); view.run(check=True)
            fps = graph_rounds(view, n_demo, False, step=lambda i: view.set_inputs(timestep=i % T))
        print(json.dumps({"arm": arm, "protocol": "demo", "splats": P_demo, "W": W, "H": H, "fovy_deg": 20.0,
                          "flame_timesteps": T, "timestep_advances_every_frame": True,
                          "fps_median": round(fps[1], 1), "fps_best": round(fps[2], 1),
                          "ms_median": round(1e3 / fps[1], 4), "rounds": 3, "iters_per_round": n_demo, "runs": 1,
                          **gpu_info()}), flush=True)
