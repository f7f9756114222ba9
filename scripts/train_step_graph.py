"""BASELINE.json config 3 (bound avatar, 150k splats, 16 cameras, --bind_to_mesh training step): one full reference
training iteration per step (train.py:106-210) -- xyz learning-rate schedule, pose, face frame, fused forward,
(1-l) L1 + l (1-SSIM) + position/scale regularisers, backward down to the vertices, densification statistics
(train.py:197 + add_densification_stats) and Adam on the six splat arrays -- timed three ways:
  eager       render() + autograd, the statistics as the reference writes them (boolean-mask indexing: a nonzero()
              and with it a host wait per line), the learning rate written on the host, host-stepped Adam
  graph       GraphedFrame for frame -> backward, then the same eager statistics, host lr and host-stepped Adam
  graph_full  ONE replay of GraphedFrame(optimizer=capturable Adam with the xyz schedule, densify_stats=True)
  graph_full_percam  the graph_full iteration over 16 cameras with DISTINCT fields of view (look_at_camera at the
              orbit poses, FoV spread +-8 %): GraphedFrame(per_camera_fov=True), the FoV read on the device per replay
With a FLAME head (synthetic.flame_like_assets on the same mesh, 16 timesteps, the reference's FLAME optimizer groups
trained as with not_finetune_flame_params=False):
  eager_flame       the eager arm with the pose of select_mesh_by_timestep from the float32 reference-order
                    restatement (tests/flame_oracle.py) + autograd, and torch's Adam on the FLAME groups
  graph_full_flame  ONE replay of GraphedFrame on the FLAME model: pose, frame, statistics and Adam over the splat and
                    FLAME groups
graph_full stays beside them as the no-FLAME lower bound.
One JSON line per resolution, with the GPU it ran on and its power limit.

    python scripts/train_step_graph.py            (ITERS=256 timed steps after 8 warm-up steps; P=150000)
"""
import json, math, os, subprocess, sys
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np
import torch
import gaussianavatars_b200 as g
from gaussianavatars_b200 import synthetic as syn
from gaussianavatars_b200.graph import GraphedFrame, camera_block
from gaussianavatars_b200.model import MeshBoundGaussians
from gaussianavatars_b200.renderer import render
from tests import flame_oracle as fo

dev = torch.device("cuda:0")
class Pipe: debug = False; compute_cov3D_python = False; convert_SHs_python = False
P, K = int(os.environ.get("P", 150000)), int(os.environ.get("ITERS", 256))
verts, faces = syn.head_mesh()
params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=0, sh_degree=3)
bg = torch.ones(3, device=dev)
NAMES = ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest")   # pc.parameters() order
LRS = dict(xyz=0.0, rotation=1e-3, scaling=5e-3, opacity=5e-2, f_dc=2.5e-3, f_rest=1.25e-4)
SCHED = g.expon_lr_schedule(lr_init=5e-3, lr_final=5e-5, lr_delay_mult=0.01, max_steps=600_000)   # OptimizationParams
FLAME_ASSETS = syn.flame_like_assets(0)
FLAME_SEQ = syn.flame_like_sequence(16, seed=1, V=FLAME_ASSETS["v_template"].shape[0])
FLAME_SEQ.pop("dynamic_offset")


def xyz_lr(it):
    """The reference's exponential schedule on the host (what update_learning_rate writes every iteration)."""
    t = np.clip(it / SCHED["max_steps"], 0, 1)
    return float(np.exp(np.log(SCHED["lr_init"]) * (1 - t) + np.log(SCHED["lr_final"]) * t))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().split("\n")[0]
    return torch.cuda.get_device_name(dev), q.split(",")[-1].strip() if q else "unknown"


def reference_stats(pc, radii, vp_grad):
    vis = radii > 0   # render()'s visibility_filter
    pc.max_radii2D[vis] = torch.max(pc.max_radii2D[vis], radii[vis])
    pc.xyz_gradient_accum[vis] += torch.norm(vp_grad[vis, :2], dim=-1, keepdim=True)
    pc.denom[vis] += 1


def timed(fn):
    for i in range(8): fn(i + 1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(K): fn(9 + i)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / K


name, power = gpu_info()
for (W, H) in ((550, 802), (1920, 1080)):
    cams = [syn.orbit_camera(W, H, azimuth_deg=-60 + 120 * (i + .5) / 16, elevation_deg=5 * math.sin(i)) for i in range(16)]
    gts = [torch.randint(0, 256, (3, H, W), dtype=torch.uint8, device=dev) for _ in range(2)]
    res = {"config": "3", "splats": P, "W": W, "H": H, "timed_steps": K, "gpu": name, "power_limit": power}
    # the same poses with distinct fields of view: 20 deg vertical (the orbit default) scaled by 0.92 .. 1.08
    fov_cams = []
    for i, c in enumerate(cams):
        f = 1.0 + 0.08 * (2 * i / 15 - 1)
        fov_cams.append(syn.look_at_camera(W, H, math.degrees(c.FoVx) * f, math.degrees(c.FoVy) * f,
                                           w2c=c.world_view_transform.T.numpy()))
    for arm in ("eager", "graph", "graph_full", "graph_full_percam", "eager_flame", "graph_full_flame"):
        flame = arm.endswith("_flame")
        if flame:
            a = FLAME_ASSETS
            lbs = g.FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], a["parents"],
                                         a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
            fparam = {k: v.to(dev).clone().contiguous() for k, v in FLAME_SEQ.items()}
            pc = MeshBoundGaussians(params, 3, None, None, device=dev, requires_grad=True, flame=lbs, flame_param=fparam)
        else:
            pc = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=dev, requires_grad=True)
        pc.xyz_gradient_accum = torch.zeros((P, 1), device=dev)
        pc.denom = torch.zeros((P, 1), device=dev)
        pc.max_radii2D = torch.zeros((P,), device=dev)
        groups = [{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(NAMES, pc.parameters())]
        if arm.startswith("graph_full"):
            groups[0]["lr_schedule"] = SCHED
        if arm == "graph_full_flame":
            groups += g.flame_param_groups(pc.flame_param)
        opt = g.Adam(groups, lr=0.0, eps=1e-15, capturable=arm.startswith("graph_full"))
        posed = None if flame else [syn.pose_mesh(pc.verts_rest, i).contiguous() for i in range(16)]
        if arm == "eager_flame":
            cd = [c.to(dev) for c in cams]
            oa = fo.assets_as({k: FLAME_ASSETS[k] for k in ("v_template", "shapedirs", "posedirs", "J_regressor",
                                                            "lbs_weights")} | {"parents": FLAME_ASSETS["parents"].tolist()},
                              torch.float32, dev)
            opt_f = torch.optim.Adam(g.flame_param_groups(pc.flame_param), lr=0.0, eps=1e-15)
            def step(it):
                opt.param_groups[0]["lr"] = xyz_lr(it)
                opt.zero_grad(set_to_none=True)
                opt_f.zero_grad(set_to_none=True)
                v, pc.verts_cano, _ = fo.select_mesh_by_timestep(oa, pc.flame_param, it % 16)
                pc.update_mesh_properties(v[0])
                out = render(cd[it % 16], pc, Pipe, bg)
                loss = g.photometric_loss(out["render"], gts[it % 2], 0.2)
                lx, ls = g.binding_regularizers(pc._xyz, pc._scaling, out["radii"], pc.binding, pc.face_scaling)
                (loss + lx + ls).backward()
                reference_stats(pc, out["radii"], out["viewspace_points"].grad)
                opt.step()
                opt_f.step()
        elif arm == "eager":
            cd = [c.to(dev) for c in cams]
            def step(it):
                opt.param_groups[0]["lr"] = xyz_lr(it)
                opt.zero_grad(set_to_none=True)
                v = posed[it % 16].requires_grad_(True)
                pc.update_mesh_properties(v)
                out = render(cd[it % 16], pc, Pipe, bg)
                loss = g.photometric_loss(out["render"], gts[it % 2], 0.2)
                lx, ls = g.binding_regularizers(pc._xyz, pc._scaling, out["radii"], pc.binding, pc.face_scaling)
                (loss + lx + ls).backward()
                reference_stats(pc, out["radii"], out["viewspace_points"].grad)
                opt.step()
        else:
            percam = arm == "graph_full_percam"
            blocks = [camera_block(c, fov=True).to(dev) for c in fov_cams] if percam else \
                [camera_block(c).to(dev) for c in cams]
            kw = dict(optimizer=opt, densify_stats=True) if arm.startswith("graph_full") else {}
            fr = GraphedFrame(pc, W, H, cams[0].FoVx, cams[0].FoVy, bg, loss="photometric", lambda_dssim=0.2,
                              regularizers={}, warm_cameras=blocks, per_camera_fov=percam, **kw)
            if flame:
                fr.set_inputs(camera=blocks[0], timestep=0, gt_u8=gts[0])
            else:
                fr.set_inputs(camera=blocks[0], verts=posed[0], gt_u8=gts[0])
            fr.capture()
            if arm == "graph":
                def step(it):
                    opt.param_groups[0]["lr"] = xyz_lr(it)
                    fr.set_inputs(camera=blocks[it % 16], verts=posed[it % 16], gt_u8=gts[it % 2])
                    fr.run()
                    reference_stats(pc, fr.radii, fr.viewspace_points.grad)
                    opt.step()
            elif flame:
                def step(it):
                    fr.set_inputs(camera=blocks[it % 16], timestep=it % 16, gt_u8=gts[it % 2])
                    fr.run()
            else:
                def step(it):
                    fr.set_inputs(camera=blocks[it % 16], verts=posed[it % 16], gt_u8=gts[it % 2])
                    fr.run()
        res[arm + "_ms_per_step"] = round(timed(step), 4)
        if arm.startswith("graph"):
            res[arm + "_overflow"] = fr.overflowed()
            res[arm + "_captures"] = fr.captures
            res[arm + "_loss_finite"] = bool(torch.isfinite(fr.loss))
        res[arm + "_denom_max"] = float(pc.denom.max())
    print(json.dumps(res), flush=True)
