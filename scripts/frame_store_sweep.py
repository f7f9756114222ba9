"""What holding the training frames in the device frame store costs and saves -> one JSON line per measurement on
stdout (profiles/h100/frame_store.jsonl):

  decode      gab200_frame_decode alone: CUDA events around 200 launches of K views, per view, and the bytes it moves
              (the records it reads plus 4 B written per pixel) over that time.  Frames: avatar renders and noise.
  iteration   per-view time of the captured FLAME training iteration (GraphedFrame: pose + render + photometric loss +
              regularisers + backward + densification statistics + capturable Adam), two arms:
                (a) rgba_pair  rgba=True, the RGBA frames copied from a pinned host cache into the staging tensors of a
                               prefetching pair of frames (host_inputs=True), whose graphs upload them for each other
                (b) store      frames=store: set_inputs(camera table already on the device, timestep, K ids), the
                               graph decodes gt and mask
              A pass is 16 cameras x 2 FLAME timesteps = 32 views, K views per replay; the arms alternate pass by pass,
              5 passes each after a warm-up pass; median, min and max.  `host_ms_per_iter` is the host time spent
              enqueueing one iteration (set_inputs / staging writes / run), median over the passes.
  encode      FrameStore.add of 16 frames (plan, one synchronisation, encode): frames per second, median of 5.
  ratio       raw bytes / stored bytes (records + index) for noise frames (the worst case) and for frames rendered
              from the synthetic avatar with its alpha plane as the mask.  The synthetic renders are smoother than
              real captures: the ratio on real captures is not measured here.

Settings: the demo (550x802, 89,021 splats) and 100k splats at 1920x1080, K in {1, 16}.  Every line carries the card,
its power limit and its SM clock, read in the same run."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import gaussianavatars_b200 as g  # noqa: E402
from gaussianavatars_b200.graph import GraphedFrame, camera_block  # noqa: E402
from gaussianavatars_b200.renderer import render  # noqa: E402
from scripts.rgba_mask_sweep import rgba_frames  # noqa: E402
from scripts.train_views_sweep import gpu_info, setting, timed  # noqa: E402

dev = torch.device("cuda:0")
STEPS = (0, 5)
VIEWS = 16 * len(STEPS)
PASSES = 5


class _Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def avatar_frames(pc, cams, H, W):
    """(16,3,H,W) uint8 renders of the synthetic avatar over white and their (16,1,H,W) alpha planes as the mask."""
    gts, masks = [], []
    bg = torch.ones(3, device=dev)
    with torch.no_grad():
        for i, cam in enumerate(cams):
            pc.select_mesh_by_timestep(i % 8)
            out = render(cam, pc, _Pipe, bg, depth_alpha=True)
            gts.append((out["render"] * 255 + 0.5).clamp(0, 255).to(torch.uint8))
            masks.append((out["alpha"] * 255 + 0.5).clamp(0, 255).to(torch.uint8))
    return torch.stack(gts), torch.stack(masks)


def decode_lines(name, store, ids_of, H, W, info, frames):
    out = []
    for K in (1, 16):
        ids = torch.tensor(ids_of(K), dtype=torch.int32, device=dev)
        gt = torch.empty((K, 3, H, W), dtype=torch.uint8, device=dev)
        mask = torch.empty((K, 1, H, W), dtype=torch.uint8, device=dev)
        for _ in range(10):
            store.launch_decode(ids, gt, mask)
        n = 200

        def many():
            for _ in range(n):
                store.launch_decode(ids, gt, mask)
        ms = sorted(timed(many) for _ in range(5))
        us = ms[2] * 1e3 / n
        fb = store.frame_base.cpu().tolist() + [store._used]
        read = sum(fb[i + 1] - fb[i] for i in ids.tolist()) + K * (8 + 4 * store.n_tiles)
        moved = read + 4 * K * H * W
        out.append(dict(setting=name, W=W, H=H, K=K, arm="decode", frames=frames, launches=n,
                        us_per_launch_median=round(us, 3), us_per_view_median=round(us / K, 3),
                        us_per_view_min=round(ms[0] * 1e3 / n / K, 3), us_per_view_max=round(ms[-1] * 1e3 / n / K, 3),
                        bytes_read_per_launch=read, bytes_per_launch=moved,
                        GB_per_s=round(moved / (us * 1e-6) / 1e9, 1), **info))
    return out


def iteration_arms(pc, opt, cams, rgba_pinned, store, W, H, K):
    groups = [cams[i:i + K] for i in range(0, 16, K)]
    warm = groups if K > 1 else cams
    kw = dict(loss="photometric", regularizers={}, optimizer=opt, densify_stats=True, per_camera_fov=True,
              views_per_replay=K, warm_cameras=warm)
    pair = [GraphedFrame(pc, W, H, 1.0, 1.0, torch.ones(3), host_inputs=True, rgba=True, **kw) for _ in range(2)]
    pair[0].prefetch_for(pair[1])
    pair[1].prefetch_for(pair[0])
    st = GraphedFrame(pc, W, H, 1.0, 1.0, torch.ones(3), frames=store, **kw)
    host = {"rgba_pair": [], "store": []}
    blocks = [torch.stack([camera_block(c, fov=True) for c in grp]).cpu().reshape(pair[0].cam_stage.shape)
              for grp in groups]
    work = [(t, j) for t in STEPS for j in range(len(groups))]

    def stage(fr, i):
        t, j = work[i]
        fr.cam_stage.copy_(blocks[j])
        fr.gt_stage.copy_(rgba_pinned[j * K:(j + 1) * K].reshape(fr.gt_stage.shape))
        fr.timestep.fill_(t)   # a device int (fill: no host wait); ordered before the replay on the main stream

    def run_pair():
        t0 = time.perf_counter()
        events = [None, None]
        stage(pair[0], 0)
        pair[0].upload_staged()
        for i in range(len(work)):
            cur, nxt = pair[i % 2], pair[(i + 1) % 2]
            if i + 1 < len(work):
                if events[i % 2] is not None:   # nxt's stage was last copied by cur's graph, in replay i - 2
                    events[i % 2].synchronize()
                stage(nxt, i + 1)
            cur.run()
            ev = torch.cuda.Event()
            ev.record()
            events[i % 2] = ev
        host["rgba_pair"].append((time.perf_counter() - t0) * 1e3 / len(work))

    tables = [b.to(dev) for b in blocks]   # the same camera blocks, already on the device

    def run_store():
        t0 = time.perf_counter()
        for t, j in work:
            ids = list(range(j * K, (j + 1) * K))
            if K > 1:
                st.set_inputs(cameras=tables[j], timestep=t, frames=ids)
            else:
                st.set_inputs(camera=tables[j], timestep=t, frames=ids[0])
            st.run()
        host["store"].append((time.perf_counter() - t0) * 1e3 / len(work))
    return {"rgba_pair": run_pair, "store": run_store}, pair + [st], host


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    for name, P, W, H in (("demo", 89_021, 550, 802), ("1080p", 100_000, 1920, 1080)):
        pc, opt, cams, _ = setting(P, W, H)
        bg = [1.0, 1.0, 1.0]
        # compression and encode throughput: avatar renders and noise
        gts, masks = avatar_frames(pc, cams, H, W)
        noise = torch.randint(0, 256, (16, 4, H, W), generator=torch.Generator().manual_seed(2),
                              dtype=torch.uint8).to(dev)
        stores = {}
        for kind, (gt, mask) in (("avatar", (gts, masks)), ("noise", (noise[:, :3].contiguous(),
                                                                       noise[:, 3:].contiguous()))):
            ts = []
            for rep in range(5):
                s = g.FrameStore(W, H, bg, dev)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                s.add(gt, mask)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            ts.sort()
            stores[kind] = s
            emit(dict(setting=name, W=W, H=H, arm="encode", frames=kind, n=16, frames_per_s_median=round(16 / ts[2], 1),
                      frames_per_s_min=round(16 / ts[-1], 1), frames_per_s_max=round(16 / ts[0], 1), **info))
            emit(dict(setting=name, W=W, H=H, arm="ratio", frames=kind, n=16, raw_bytes=s.raw_nbytes,
                      stored_bytes=s.nbytes, ratio=round(s.raw_nbytes / s.nbytes, 3),
                      bound_bytes=16 * (s.n_tiles * 1036 + 8), synthetic=True, **info))
        for kind, s in stores.items():
            for rec in decode_lines(name, s, lambda K: list(range(K)), H, W, info, kind):
                emit(rec)
        # the captured iteration: RGBA through a prefetching pair vs the store
        rgba = rgba_frames(16, H, W)
        rgba_pinned = rgba.pin_memory()
        store = g.FrameStore(W, H, bg, dev)
        store.add_rgba(rgba.to(dev))
        for K in (1, 16):
            fns, frames, host = iteration_arms(pc, opt, cams, rgba_pinned, store, W, H, K)
            for fn in fns.values():   # warm-up pass (captures)
                fn()
            torch.cuda.synchronize()
            for v in host.values():
                v.clear()
            ms = {k: [] for k in fns}
            for _ in range(PASSES):
                for k, fn in fns.items():
                    ms[k].append(timed(fn))
            overflow = any(f.overflowed() for f in frames)
            for arm, v in ms.items():
                v, hv = sorted(v), sorted(host[arm])
                emit({"setting": name, "splats": P, "W": W, "H": H, "K": K, "arm": arm, "views_per_pass": VIEWS,
                      "ms_per_view_median": round(v[len(v) // 2] / VIEWS, 4), "ms_per_view_min": round(v[0] / VIEWS, 4),
                      "ms_per_view_max": round(v[-1] / VIEWS, 4), "host_ms_per_iter_median": round(hv[len(hv) // 2], 4),
                      "passes": len(v), "overflow": overflow, "captures": [f.captures for f in frames], **info})
            del fns, frames
            torch.cuda.empty_cache()
        del pc, opt, stores, store
        torch.cuda.empty_cache()
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
