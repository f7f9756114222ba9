"""Per-view cost of the tracked mesh over every camera of a K-view replay (gab200_mesh_render_views) -> one JSON line
per (setting, arm) on stdout (kept in profiles/h100/mesh_views.jsonl):

  render_views_mesh    GraphedRender(views_per_replay=K, mesh_opacity=0.5): pose, K-view splat forward, one K-view
                       mesh overlay -- K in {1, 4, 16}, ms per view = replay / K
  render_single_mesh   the same K cameras as K single-view GraphedRender(mesh_opacity=0.5) replays
  eval_scheduled_mesh  a scheduled GraphedEval(source="u8", mesh_opacity=0.5, png=True) over a set (render.py's renders,
                       renders_mesh, both PNG sets and the scores, no host input), K = 1 and 4
  eval_eager_mesh      the same set scored by a scheduled GraphedEval(png=True), then per view the posed vertices, the
                       decoded ground truth, an eager mesh_overlay(base=gt) and encode_png (render.py's loop today)

Protocol: a warm-up pass, then 3 timed passes, CUDA events around each (the eval arms end in a synchronise), the
median pass reported per view.  100k splats on the 9,996-face head, orbit cameras around it at 550x802 and 1920x1080.
Every line carries the card and its power limit, read in the same run.

    python scripts/mesh_views_sweep.py                        # the sweep, on the GPU
    python scripts/mesh_views_sweep.py --sizes 64x48 --ks 1,2 --records 4 --splats 1000   # a rehearsal

The plan (settings, views, the K-view scratch from gab200_mesh_views_scratch_bytes) is printed before any device
work, so a rehearsal without a GPU checks arguments and shapes and stops at the first device call."""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

from gaussianavatars_b200 import _native as N  # noqa: E402

PASSES = 3
FACES = 9996   # the synthetic FLAME-like head's


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="550x802,1920x1080", help="WxH settings, comma-separated")
    ap.add_argument("--ks", default="1,4,16", help="views per replay of the render arms")
    ap.add_argument("--eval-ks", default="1,4", help="views per replay of the eval arms")
    ap.add_argument("--records", type=int, default=32, help="views in the eval set (records x K)")
    ap.add_argument("--replays", type=int, default=20, help="K-view replays per timed render pass")
    ap.add_argument("--splats", type=int, default=100_000)
    a = ap.parse_args(argv)
    a.sizes = [tuple(int(x) for x in s.lower().split("x")) for s in a.sizes.split(",")]
    a.ks = [int(k) for k in a.ks.split(",")]
    a.eval_ks = [int(k) for k in a.eval_ks.split(",")]
    for k in a.ks + a.eval_ks:
        if not 1 <= k <= N.MAX_VIEWS:
            raise SystemExit(f"views per replay must lie in [1, {N.MAX_VIEWS}], got {k}")
    for k in a.eval_ks:
        if a.records % k:
            raise SystemExit(f"--records {a.records} is not a multiple of K = {k}")
    return a


def plan(a):
    """One line per setting: the views timed and the K-view overlay's scratch (no device needed)."""
    L = N.lib()
    for W, H in a.sizes:
        scratch = {k: int(L.gab200_mesh_views_scratch_bytes(k, FACES, W, H)) for k in a.ks}
        yield {"plan": f"{W}x{H}", "W": W, "H": H, "render_views_per_pass": {k: k * a.replays for k in a.ks},
               "eval_views": a.records, "mesh_views_scratch_bytes": scratch}


def gpu_info(dev):
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip().split(", ")
    if len(q) != 3:
        return {"gpu": torch.cuda.get_device_name(dev)}
    return {"gpu": q[0], "power_limit_W": float(q[1]), "sm_clock_max_MHz": float(q[2])}


def model(dev, P, T=8):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.flame import FlameLBS
    from gaussianavatars_b200.model import MeshBoundGaussians
    a = syn.flame_like_assets(0)
    fp = {k: v.to(dev).contiguous() for k, v in syn.flame_like_sequence(T, seed=1, V=a["v_template"].shape[0]).items()
          if k != "dynamic_offset"}
    lbs = FlameLBS.from_arrays(a["v_template"], a["shapedirs"], a["posedirs"], a["J_regressor"], list(a["parents"]),
                               a["lbs_weights"], a["faces"], a["n_shape"], a["n_expr"], device=dev)
    params = syn.avatar_splats(P, n_faces=a["faces"].shape[0], seed=0, sh_degree=3)
    return MeshBoundGaussians(params, 3, None, None, device=dev, flame=lbs, flame_param=fp)


def cameras(W, H, n):
    from gaussianavatars_b200 import synthetic as syn
    r = 1.0 if H > W else 0.6   # the head fills a portrait frame at 1.0, a landscape one at 0.6
    return [syn.orbit_camera(W, H, r=r, fovy_deg=20.0, azimuth_deg=-40 + 80 * i / max(n - 1, 1),
                             elevation_deg=5 * math.sin(i)) for i in range(n)]


def timed(step, n):
    """n calls per pass after a warm-up pass; sorted per-pass ms."""
    for i in range(n):
        step(i)
    torch.cuda.synchronize()
    ms = []
    for _ in range(PASSES):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            step(i)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return sorted(ms)


def render_arms(pc, W, H, ks, replays, bg):
    from gaussianavatars_b200.graph import GraphedRender
    for K in ks:
        cams = cameras(W, H, K)
        view = GraphedRender(pc, W, H, bg, outputs="u8", views_per_replay=K, mesh_opacity=0.5,
                             warm_cameras=[cams] if K > 1 else cams, warm_timesteps=range(8))

        group = dict(cameras=cams) if K > 1 else dict(camera=cams[0])

        def many(i, view=view, group=group):
            view.set_inputs(timestep=i % 8, **group)
            view.run()

        single = GraphedRender(pc, W, H, bg, outputs="u8", mesh_opacity=0.5, warm_cameras=cams,
                               warm_timesteps=range(8))

        def one(i, view=single, cams=cams):
            for c in cams:
                view.set_inputs(camera=c, timestep=i % 8)
                view.run()

        for arm, fn, v in (("render_views_mesh", many, view), ("render_single_mesh", one, single)):
            ms = timed(fn, replays)
            assert not v.overflowed() and v.captures == 1 and int(v.mesh_error.item()) == 0
            yield {"arm": arm, "K": K, "views_per_pass": K * replays,
                   "ms_per_view_median": round(ms[1] / (K * replays), 4),
                   "ms_per_view_best": round(ms[0] / (K * replays), 4)}
        del view, single
        torch.cuda.empty_cache()


def eval_arms(pc, W, H, ks, records, bg, dev):
    from gaussianavatars_b200 import FrameStore, ViewSchedule, encode_png, mesh_overlay
    from gaussianavatars_b200.graph import GraphedEval
    gen = torch.Generator().manual_seed(3)
    for K in ks:
        R = records // K
        cams = cameras(W, H, records)
        groups = [cams[r * K:(r + 1) * K] for r in range(R)]
        ts = [r % 8 for r in range(R)]
        store = FrameStore(W, H, bg.cpu(), dev)
        rgba = torch.randint(0, 256, (records, H, W, 4), generator=gen, dtype=torch.uint8)
        rgba[..., 3] = 255
        store.add_rgba(rgba)
        del rgba
        ids = [[r * K + k for k in range(K)] for r in range(R)]
        s = ViewSchedule([g[0] for g in groups] if K == 1 else groups, timesteps=ts,
                         frames=[i[0] for i in ids] if K == 1 else ids, device=dev)
        common = dict(views=records, source="u8", views_per_replay=K, schedule=s, frames=store, png=True)
        ea = GraphedEval(pc, W, H, bg, mesh_opacity=0.5, **common)
        eb = GraphedEval(pc, W, H, bg, **common)

        def scheduled(i):
            ea.reset()
            assert ea.run_all(check=True) == R

        def eager(i):
            eb.reset()
            assert eb.run_all(check=True) == R
            for r in range(R):
                gt, _ = store.decode(ids[r])
                pc.select_mesh_by_timestep(ts[r])
                for k in range(K):
                    encode_png(mesh_overlay(pc.verts, pc.faces, groups[r][k], gt[k]))

        for arm, fn in (("eval_scheduled_mesh", scheduled), ("eval_eager_mesh", eager)):
            ms = timed(fn, 1)
            yield {"arm": arm, "K": K, "views_per_pass": records, "ms_per_view_median": round(ms[1] / records, 4),
                   "ms_per_view_best": round(ms[0] / records, 4)}
        assert ea.captures == 1 and int(ea.mesh_error.item()) == 0
        del ea, eb, store, s
        torch.cuda.empty_cache()


def main(argv=None):
    a = parse(argv)
    plans = list(plan(a))
    for p in plans:
        print(json.dumps(p), flush=True)
    if not torch.cuda.is_available():
        raise SystemExit("mesh_views_sweep: no CUDA device -- the plan above is all a run without a GPU gives")
    dev = torch.device("cuda:0")
    info = gpu_info(dev)
    pc = model(dev, a.splats)
    bg = torch.ones(3, device=dev)
    for (W, H), p in zip(a.sizes, plans):
        lines = list(render_arms(pc, W, H, a.ks, a.replays, bg)) + \
            list(eval_arms(pc, W, H, a.eval_ks, a.records, bg, dev))
        for line in lines:
            scratch = p["mesh_views_scratch_bytes"].get(line["K"])
            line.update({"setting": f"{W}x{H}", "W": W, "H": H, "splats": int(pc._xyz.shape[0]),
                         "faces": int(pc.faces.shape[0]), "passes": PASSES, **info})
            if scratch is not None:
                line["mesh_views_scratch_bytes"] = scratch
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
