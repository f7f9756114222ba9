"""GPU: the K-view mesh overlay (gab200_mesh_render_views, mesh_overlay_views) and the replays that draw it.

  * the kernels: every output of one K-view call -- the out_u8 planes and the error flag -- equals K calls of
    gab200_mesh_render byte for byte, K in {1, 2, 5, 16}, on the cameras of tests/test_gpu_mesh.py (orbit views, a
    close-up whose largest face covers ~1.5e5 px and crosses the near plane, a camera inside the head, a grazing
    view) mixed in one call and repeated, on the rigs of tests/bound_rigs.py, over float and uint8 bases, with face
    colours, both lightings and antialias off; a spot check against tests/mesh_oracle.py; an out-of-range face index;
  * GraphedRender(views_per_replay=K, mesh_opacity=): each replay's display is render_views then mesh_overlay per
    view; a new opacity or new face colours never re-capture; the PNG files and the host slots carry the frames;
  * scheduled GraphedEval(mesh_opacity=0.5, png=True, host_slots=2) at K = 1 and 4 over 16 records: mesh_display is
    mesh_overlay of the record's posed vertices, cameras and decoded ground truth; scores, display and render PNGs are
    those of the same GraphedEval without the mesh; the mesh PNGs decode to mesh_display; a VideoWriter fed
    mesh_display writes encode_video's bytes; an overflowed replay still draws and ships its mesh frame."""
import io

import numpy as np
import pytest
import torch

from gaussianavatars_b200 import mesh_overlay, mesh_overlay_views
from gaussianavatars_b200 import synthetic as syn
from gaussianavatars_b200.graph import camera_block
from gaussianavatars_b200.mesh import launch_mesh, mesh_adjacency, opacity_pair
from gaussianavatars_b200.renderer import camera_table
from tests import bound_rigs as B
from tests import mesh_oracle as mo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
W_M, H_M = 550, 802

# the camera kinds of tests/test_gpu_mesh.py, at one image size (a K-view call has one)
KINDS = {
    "orbit": dict(r=1.0, az=25.0, el=0.0),
    "orbit_high": dict(r=0.6, az=-40.0, el=10.0),
    "orbit_low": dict(r=0.7, az=70.0, el=-15.0),
    "closeup_near_plane": dict(r=0.1147, az=90.0, el=0.0),
    "inside_head": dict(r=0.0, az=0.0, el=0.0, fovy=60.0),
    "grazing": dict(r=0.8, az=10.0, el=84.0),
}
# K -> the kinds of the call's views, in order: every kind mixed, and repeated cameras
RIGS = {
    1: ["closeup_near_plane"],
    2: ["inside_head", "grazing"],
    5: ["orbit", "closeup_near_plane", "inside_head", "grazing", "orbit"],
    16: [list(KINDS)[i % len(KINDS)] for i in range(15)] + ["closeup_near_plane"],
}
VARIANTS = {
    "u8": dict(),
    "float_base": dict(base="float"),
    "colors_constant": dict(colors=True, lighting="constant"),
    "colors_front_no_aa": dict(colors=True, antialias=False),
}


def _camera(kind, W=W_M, H=H_M):
    s = KINDS[kind]
    return syn.orbit_camera(W, H, r=s["r"], fovy_deg=s.get("fovy", 20.0), azimuth_deg=s["az"], elevation_deg=s["el"])


def _head():
    verts, faces = syn.head_mesh(seed=0)
    return torch.tensor(np.asarray(verts, np.float32), device=DEV), torch.tensor(np.asarray(faces), device=DEV)


def _bases(K, W, H, kind, seed=1):
    u8 = torch.randint(0, 256, (K, 3, H, W), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)
    return (u8.float() / 255 if kind == "float" else u8).to(DEV)


def _both(verts, faces, table, base, colors=None, lighting="front", antialias=True, opacity=0.5):
    """(K-view call, K single-view calls): (out_u8 (K,H,W,3), error flag) each."""
    K, _, H, W = base.shape
    f = faces.to(torch.int32).contiguous()
    common = dict(verts=verts, faces=f, width=W, height=H, adjacency=mesh_adjacency(f) if antialias else None,
                  face_colors=colors, lighting=lighting, antialias=antialias, opacity=opacity_pair(opacity, DEV))
    many, flag_many = torch.full((K, H, W, 3), 7, dtype=torch.uint8, device=DEV), torch.zeros(1, dtype=torch.int32,
                                                                                                device=DEV)
    launch_mesh(camera=table, base=base, out_u8=many, error_flag=flag_many, views=K, **common)
    one, flag_one = torch.full((K, H, W, 3), 9, dtype=torch.uint8, device=DEV), torch.zeros(1, dtype=torch.int32,
                                                                                              device=DEV)
    for k in range(K):
        launch_mesh(camera=table[k].contiguous(), base=base[k].contiguous(), out_u8=one[k], error_flag=flag_one,
                    **common)
    torch.cuda.synchronize()
    return (many, int(flag_many.item())), (one, int(flag_one.item()))


# ---- the kernels -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("K", sorted(RIGS))
def test_views_equal_single_view_calls_byte_for_byte(K, variant):
    v, f = _head()
    opt = VARIANTS[variant]
    cams = [_camera(k) for k in RIGS[K]]
    table = camera_table(cams, DEV)
    base = _bases(K, W_M, H_M, opt.get("base"), seed=K)
    colors = torch.rand(f.shape[0], 3, generator=torch.Generator().manual_seed(3)).to(DEV) if opt.get("colors") \
        else None
    (many, flag_many), (one, flag_one) = _both(v, f, table, base, colors=colors, lighting=opt.get("lighting", "front"),
                                               antialias=opt.get("antialias", True))
    for k in range(K):
        assert torch.equal(many[k], one[k]), f"view {k} ({RIGS[K][k]}): " \
            f"{int((many[k] != one[k]).any(-1).sum())} pixels differ"
    assert flag_many == flag_one == 0
    # the mesh is drawn in every view (not just the base), and differently per kind
    plain = base if base.dtype == torch.uint8 else base.mul(255).add(0.5).clamp(0, 255).to(torch.uint8)
    for k in range(K):
        assert (many[k].permute(2, 0, 1) != plain[k]).any(0).float().mean() > 0.005, f"view {k}: no mesh"
    if K >= 5:
        assert not torch.equal(many[0], many[1])


@pytest.mark.parametrize("name", ["needles", "near_plane", "guard_band"])
def test_bound_rigs_equal_single_view_calls(name):
    from tests.test_oracle_multiview_adversarial import scene
    bound = B.bind(scene((name, None, None)))
    cams = B.rig(bound, 6)
    table = B.table(cams, DEV)   # row 5's field of view is invalid: the mesh reads only the two matrices
    v = torch.as_tensor(np.asarray(bound["verts"], np.float32), device=DEV)
    f = torch.as_tensor(np.asarray(bound["faces"], np.int64), device=DEV)
    for base_kind in ("u8", "float"):
        base = _bases(6, bound["W"], bound["H"], base_kind, seed=5)
        (many, flag_many), (one, flag_one) = _both(v, f, table, base)
        assert torch.equal(many, one), f"{name} {base_kind}"
        assert flag_many == flag_one == 0


def test_a_subset_against_the_oracle():
    v, f = _head()
    kinds = ["orbit", "closeup_near_plane", "grazing"]
    cams = [_camera(k) for k in kinds]
    base = _bases(3, W_M, H_M, "u8", seed=11)
    colors = np.random.default_rng(2).random((f.shape[0], 3)).astype(np.float32)
    got = mesh_overlay_views(v, f, cams, base, face_colors=torch.tensor(colors, device=DEV)).cpu().numpy()
    faces = f.cpu().numpy()
    adj = mesh_adjacency(f.cpu()).numpy()
    for k, cam in enumerate(cams):
        m = mo.Mesh(faces, W_M, H_M, verts=v.cpu().numpy(), block=camera_block(cam).numpy(), face_colors=colors)
        ref = mo.quantize(mo.composite(m.rgba(adj), base[k].cpu().numpy(), 0.5))
        assert (got[k] == ref).all(), f"{kinds[k]}: {int((got[k] != ref).any(-1).sum())} pixels differ"
        if kinds[k] == "closeup_near_plane":
            fid = m.face_id
            assert np.bincount(fid[fid >= 0]).max() >= 100_000


def test_bad_face_index_sets_the_flag_in_every_view():
    v, f = _head()
    bad = f.clone()
    bad[100] = torch.tensor([0, 1, v.shape[0] + 7])
    bad[200] = torch.tensor([-3, 1, 2])
    cams = [_camera(k) for k in ("orbit", "grazing", "orbit_high")]
    base = _bases(3, W_M, H_M, "u8", seed=4)
    (many, flag_many), (one, flag_one) = _both(v, bad, camera_table(cams, DEV), base)
    assert flag_many == flag_one == 1
    assert torch.equal(many, one)
    m = mo.Mesh(bad.cpu().numpy(), W_M, H_M, verts=v.cpu().numpy(), block=camera_block(cams[1]).numpy())
    assert not ((m.face_id == 100) | (m.face_id == 200)).any()
    ref = mo.quantize(mo.composite(m.rgba(mo.adjacency_loop(bad.cpu().numpy())), base[1].cpu().numpy(), 0.5))
    assert (many[1].cpu().numpy() == ref).all()


def test_mesh_overlay_views_equals_mesh_overlay_per_view():
    v, f = _head()
    cams = [_camera(k) for k in ("orbit", "inside_head", "orbit", "grazing")]
    base = _bases(4, W_M, H_M, "float", seed=8)
    base[2] = base[0]                    # view 2 repeats view 0: camera and base
    got = mesh_overlay_views(v, f, camera_table(cams, DEV), base, mesh_opacity=0.3, lighting="constant")
    for k, cam in enumerate(cams):
        assert torch.equal(got[k], mesh_overlay(v, f, cam, base[k], mesh_opacity=0.3, lighting="constant"))
    assert torch.equal(got[0], got[2])   # a repeated camera draws the same frame


# ---- GraphedRender(views_per_replay=K, mesh_opacity=) ---------------------------------------------------------------
def _decode(data: bytes) -> torch.Tensor:
    from PIL import Image
    return torch.from_numpy(np.asarray(Image.open(io.BytesIO(data)).convert("RGB")).copy())


def test_graphed_render_views_with_the_mesh_equals_render_views_then_mesh_overlay():
    from gaussianavatars_b200.graph import GraphedRender
    from gaussianavatars_b200.renderer import render_views
    from tests.test_gpu_display import H_IMG, W_IMG, Pipe, _flame_setup, _rig
    K = 4
    pc = _flame_setup()
    cams = _rig(W_IMG, H_IMG, n=K)
    bg = torch.tensor([1.0, 1.0, 1.0])
    F = pc.faces.shape[0]
    colors = torch.rand(F, 3, generator=torch.Generator().manual_seed(7)).to(DEV)
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", views_per_replay=K, warm_cameras=[cams, cams[::-1]],
                         warm_timesteps=range(8), mesh_opacity=0.5, face_colors=colors, host_slots=2, png=True)
    checks = [(0, 0.5, None, cams), (3, 0.5, None, cams[::-1]), (5, 0.8, torch.rand(F, 3).to(DEV), cams),
              (6, 0.25, torch.rand(1, F, 3).to(DEV), cams)]
    for i, (t, o, new_colors, group) in enumerate(checks):
        if new_colors is not None:
            colors = new_colors.reshape(F, 3)
        view.set_inputs(cameras=group, timestep=t, mesh_opacity=o, face_colors=new_colors)
        view.run(check=True)
        torch.cuda.synchronize()
        display = view.display.clone()
        assert tuple(display.shape) == (K, H_IMG, W_IMG, 3)
        pc.select_mesh_by_timestep(t)
        ref = render_views([c.to(DEV) for c in group], pc, Pipe, bg.to(DEV), float_image=True)
        torch.cuda.synchronize()
        assert torch.equal(view.image, ref["render"])
        eager = mesh_overlay_views(pc.verts, pc.faces, group, ref["render"], mesh_opacity=o, face_colors=colors)
        assert torch.equal(display, eager), f"replay {i}"
        for k in range(K):
            want = mesh_overlay(pc.verts, pc.faces, group[k], ref["render"][k], mesh_opacity=o, face_colors=colors)
            assert torch.equal(display[k], want), f"replay {i}, view {k}"
            assert not torch.equal(want, ref["display_u8"][k])   # the mesh is on
        files = view.host_png(i)
        assert len(files) == K
        for k in range(K):
            assert torch.equal(_decode(files[k]), display[k].cpu()), f"replay {i}, view {k}"
        assert torch.equal(view.host_frame(i), display.cpu())
    assert view.captures == 1
    assert int(view.mesh_error.item()) == 0


# ---- scheduled GraphedEval(mesh_opacity=0.5, png=True) ---------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 4])
def test_scheduled_eval_draws_renders_mesh_over_the_ground_truth(K):
    from gaussianavatars_b200 import VideoWriter, encode_video
    from gaussianavatars_b200.graph import GraphedEval
    from tests import test_gpu_multiview_train as MV
    from tests.test_gpu_schedule import H_S, W_S, _records, _schedule
    R = 16
    groups, ts, ids, store = _records(R, K, seed=40 + K)
    s = _schedule(groups, ts, ids, K, None)
    pc, _ = MV._flame_trainable()
    common = dict(views=R * K, source="u8", views_per_replay=K, schedule=s, frames=store, png=True, host_slots=2)
    ea = GraphedEval(pc, W_S, H_S, torch.ones(3), mesh_opacity=0.5, **common)
    eb = GraphedEval(pc, W_S, H_S, torch.ones(3), **common)
    shown, buf = [], io.BytesIO()
    with VideoWriter(buf, W_S, H_S, fps=25, qp=20, batch=4) as vw:
        for r in range(R):
            for ev in (ea, eb):
                ev.run()
            vw.add(ea.mesh_display)
            torch.cuda.synchronize()
            got = ea.mesh_display.clone()
            shown.append(got.reshape(K, H_S, W_S, 3))
            assert torch.equal(ea.display, eb.display), f"record {r}: display changed with the mesh"
            assert ea.host_png(r) == eb.host_png(r), f"record {r}: render PNG changed with the mesh"
            gt, _ = store.decode(ids[r])
            pc.select_mesh_by_timestep(ts[r])
            want = torch.stack([mesh_overlay(pc.verts, pc.faces, groups[r][k], gt[k]) for k in range(K)])
            assert torch.equal(got.reshape(K, H_S, W_S, 3), want), f"record {r}"
            files = ea.host_mesh_png(r)
            files = [files] if K == 1 else files
            for k in range(K):
                assert torch.equal(_decode(files[k]), want[k].cpu()), f"record {r}, view {k}"
    assert int(ea.cursor) == int(eb.cursor) == R
    a, b = ea.scores(), eb.scores()
    assert torch.equal(a["per_view"], b["per_view"])
    assert ea.captures == 1 and int(ea.mesh_error.item()) == 0
    assert buf.getvalue() == encode_video(torch.cat(shown), fps=25, qp=20)


def test_an_overflowed_eval_replay_still_draws_and_ships_its_mesh_frame():
    from gaussianavatars_b200.graph import GraphedEval
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=6)
    cam = _rig(W_IMG, H_IMG, n=4)[1]
    gt = torch.randint(0, 256, (3, H_IMG, W_IMG), generator=torch.Generator().manual_seed(3), dtype=torch.uint8)
    ev = GraphedEval(pc, W_IMG, H_IMG, torch.ones(3), views=1, source="u8", host_slots=2, png=True, capacity=2000,
                     mesh_opacity=0.5)
    ev.set_inputs(camera=cam, timestep=1, gt_u8=gt, view=0)
    ev.run(check=False)
    assert ev.overflowed()
    pc.select_mesh_by_timestep(1)
    want = mesh_overlay(pc.verts, pc.faces, cam, gt.to(DEV))
    assert torch.equal(ev.mesh_display, want)
    assert torch.equal(_decode(ev.host_mesh_png(0)), want.cpu())
    with pytest.raises(RuntimeError, match="overflowed"):
        ev.host_png(0)
