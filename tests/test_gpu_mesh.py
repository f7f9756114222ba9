"""GPU: the mesh overlay kernels (csrc/mesh.cu) against their numpy restatement (tests/mesh_oracle.py) -- the winner map
at every pixel, rgba and the composite bytes bit for bit -- on orbit views up to 4K, a close-up whose faces cover more
than 1e5 pixels and cross the near plane, a camera inside the head and a grazing view; then the nvdiffrast shim driven
in the reference mesh renderer's call order, determinism, and the bad-face flag."""
import numpy as np
import pytest
import torch

from gaussianavatars_b200 import MeshRenderer, mesh_overlay
from gaussianavatars_b200 import synthetic as syn
from gaussianavatars_b200.graph import camera_block
from gaussianavatars_b200.mesh import launch_mesh, mesh_adjacency, opacity_pair
from tests import mesh_oracle as mo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

SCENES = {
    "orbit_550x802": dict(W=550, H=802, r=1.0, az=25.0, el=0.0),
    "orbit_1080p": dict(W=1920, H=1080, r=0.6, az=-40.0, el=10.0),
    "orbit_4k": dict(W=3840, H=2160, r=0.7, az=70.0, el=-15.0),
    "closeup_near_plane": dict(W=550, H=802, r=0.1147, az=90.0, el=0.0),
    "inside_head": dict(W=640, H=480, r=0.0, az=0.0, el=0.0, fovy=60.0),
    "grazing": dict(W=800, H=600, r=0.8, az=10.0, el=84.0),
}


def _scene(name, seed=0):
    s = SCENES[name]
    verts, faces = syn.head_mesh(seed=seed)
    cam = syn.orbit_camera(s["W"], s["H"], r=s["r"], fovy_deg=s.get("fovy", 20.0), azimuth_deg=s["az"],
                           elevation_deg=s["el"])
    return np.asarray(verts, np.float32), np.asarray(faces, np.int64), cam


def _gt(W, H, seed=1):
    return torch.randint(0, 256, (3, H, W), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _device_render(verts, faces, cam, gt, face_colors=None, lighting="front", opacity=0.5):
    W, H = cam.image_width, cam.image_height
    v = torch.tensor(verts, device=DEV)
    f = torch.tensor(faces, dtype=torch.int32, device=DEV)
    outs = dict(out_rast=torch.empty(H, W, 4, device=DEV), out_rgba=torch.empty(H, W, 4, device=DEV),
                out_u8=torch.empty(H, W, 3, dtype=torch.uint8, device=DEV))
    launch_mesh(verts=v, faces=f, width=W, height=H, camera=camera_block(cam).to(DEV), adjacency=mesh_adjacency(f),
                face_colors=None if face_colors is None else torch.tensor(face_colors, device=DEV),
                lighting=lighting, antialias=True, base=gt.to(DEV), opacity=opacity_pair(opacity, DEV), **outs)
    torch.cuda.synchronize()
    return {k: t.cpu().numpy() for k, t in outs.items()}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_winner_map_rgba_and_bytes_equal_the_oracle(name):
    verts, faces, cam = _scene(name)
    W, H = cam.image_width, cam.image_height
    gt = _gt(W, H)
    colors = np.random.default_rng(2).random((len(faces), 3)).astype(np.float32) if name == "grazing" else None
    got = _device_render(verts, faces, cam, gt, face_colors=colors)
    m = mo.Mesh(faces, W, H, verts=verts, block=camera_block(cam).numpy(), face_colors=colors)
    adj = mesh_adjacency(torch.tensor(faces)).numpy()
    fid = m.face_id
    covered = fid >= 0
    # kernel and oracle form the same float32 depth keys op by op, so there is no depth knife-edge to excuse: every
    # pixel is compared
    print(f"{name}: {covered.sum()} covered px, {len(np.unique(fid[covered]))} faces drawn, "
          f"largest face {np.bincount(fid[covered]).max()} px")
    if name == "closeup_near_plane":
        drawn = np.bincount(fid[covered], minlength=len(faces))
        assert drawn.max() >= 100_000
        assert drawn[m.inside != 7].max() > 0          # a face crossing the near plane is drawn
    assert (got["out_rast"][..., 3].astype(np.int64) - 1 == fid).all(), \
        f"{int((got['out_rast'][..., 3].astype(np.int64) - 1 != fid).sum())} winner pixels differ"
    rgba = m.rgba(adj)
    assert np.abs(got["out_rgba"] - rgba).max() <= 1e-6
    ref_u8 = mo.quantize(mo.composite(rgba, gt.numpy(), 0.5))
    assert (got["out_u8"] == ref_u8).all(), f"{int((got['out_u8'] != ref_u8).any(-1).sum())} pixels differ"
    assert covered.mean() > 0.01


def test_two_runs_give_identical_bytes_and_the_float_route_agrees():
    verts, faces, cam = _scene("orbit_1080p")
    gt = _gt(cam.image_width, cam.image_height).to(DEV)
    v = torch.tensor(verts, device=DEV, requires_grad=True)
    f = torch.tensor(faces, device=DEV)
    a = mesh_overlay(v, f, cam, gt)
    b = mesh_overlay(v, f, cam, gt)
    assert a.dtype == torch.uint8 and tuple(a.shape) == (cam.image_height, cam.image_width, 3)
    assert torch.equal(a, b)
    base = gt.float() / 255
    fl = mesh_overlay(v, f, camera_block(cam, fov=True), base, out="float")
    q = fl.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)
    assert torch.equal(q, a)
    assert not fl.requires_grad


def _reference_call_order(renderer_cam, verts, faces, face_colors=None, lighting="front"):
    """mesh_renderer.NVDiffRenderer.render_from_camera + render_mesh written out in the reference's order (use_opengl
    path) against the shim; returns (rast, the rgba handed to antialias, the result dict)."""
    import sys
    import os

    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "gaussianavatars_b200", "compat"))
    import nvdiffrast.torch as dr

    cam = renderer_cam
    wv = cam.world_view_transform.clone().to(verts)
    wv[:, 1] = -wv[:, 1]
    wv[:, 2] = -wv[:, 2]
    RT = wv.T[None]
    fp = cam.full_proj_transform.clone()
    fp[:, 1] = -fp[:, 1]
    full_proj = fp.T[None].to(verts)
    posw = torch.cat([verts, torch.ones([*verts.shape[:2], 1], device=verts.device)], axis=-1)
    verts_camera = torch.bmm(posw, RT.transpose(-1, -2))[..., :3]
    verts_clip = torch.bmm(posw, full_proj.transpose(-1, -2))
    image_size = cam.image_height, cam.image_width
    rast_out, _ = dr.rasterize(dr.RasterizeGLContext(), verts_clip, faces.int(), image_size)
    fg = torch.clamp(rast_out[..., -1:], 0, 1).bool()
    face_id = torch.clamp(rast_out[..., -1:].long() - 1, 0)
    i0, i1, i2 = faces[..., 0].long(), faces[..., 1].long(), faces[..., 2].long()
    v0, v1, v2 = verts_camera[..., i0, :], verts_camera[..., i1, :], verts_camera[..., i2, :]
    n = torch.cross(v1 - v0, v2 - v0, dim=-1)
    n = n / torch.sqrt(torch.clamp((n * n).sum(-1, keepdim=True), min=1e-20))
    normal = n[0][face_id[0, ..., 0]][None]
    albedo = face_colors[0][face_id[0, ..., 0]][None] if face_colors is not None else torch.ones_like(normal)
    diffuse = torch.clamp(normal[..., 2:3], 0.0, 1.0) if lighting == "front" else torch.ones_like(normal)
    rgba = torch.cat([albedo * diffuse, fg.float()], -1)
    rgba = torch.where(fg, rgba, torch.tensor([1.0, 1.0, 1.0, 0.0], device=verts.device).expand_as(rgba))
    rgba_aa = dr.antialias(rgba, rast_out, verts_clip, faces.int())
    return rast_out, verts_clip, rgba, rgba_aa.flip(1)


def test_shim_in_the_reference_call_order_matches_the_oracle_and_the_fused_renderer():
    verts, faces, cam = _scene("orbit_550x802")
    W, H = cam.image_width, cam.image_height
    v = torch.tensor(verts, device=DEV)[None].requires_grad_(True)     # as the train.py viewer passes them
    f = torch.tensor(faces, device=DEV)
    fc = torch.rand(1, len(faces), 3, generator=torch.Generator().manual_seed(4)).to(DEV)
    rast, verts_clip, rgba_in, rgba_aa = _reference_call_order(cam.to(DEV), v, f, face_colors=fc)
    assert not rast.requires_grad and not rgba_aa.requires_grad
    m = mo.Mesh(faces, W, H, pos=verts_clip[0].detach().cpu().numpy())
    assert (rast[0, ..., 3].cpu().numpy().astype(np.int64) - 1 == m.face_id).all()
    assert (rast[0, ..., 2].cpu().numpy()[m.face_id >= 0] >= -1).all()
    adj = mesh_adjacency(f).cpu().numpy()
    ref = m.antialias(rgba_in[0].detach().cpu().numpy(), adj)
    assert np.abs(rgba_aa.flip(1)[0].cpu().numpy() - ref).max() <= 1e-6
    # the barycentrics interpolate the clip position back (perspective-correct, original triangle)
    cov = rast[0, ..., 3] > 0
    fid = rast[0, ..., 3][cov].long() - 1
    u, w_ = rast[0, ..., 0][cov], rast[0, ..., 1][cov]
    tri = verts_clip[0].detach()[f.long()[fid]]
    p = u[:, None] * tri[:, 0] + w_[:, None] * tri[:, 1] + (1 - u - w_)[:, None] * tri[:, 2]
    assert torch.allclose(p[:, 2] / p[:, 3], rast[0, ..., 2][cov], atol=1e-4)
    # the fused renderer draws the same image (its own clip coordinates: ids agree away from snapping ties)
    out = MeshRenderer().render_from_camera(v, f, cam.to(DEV), face_colors=fc)
    same = (out["rgba"][0] - rgba_aa[0]).abs().amax(-1) <= 1e-5
    print(f"fused vs shim rgba: {int((~same).sum())} of {W * H} px differ")
    assert (~same).float().mean() < 1e-3
    assert out["albedo"].shape == (1, H, W, 3) and out["normal"].shape == (1, H, W, 3)


def test_bad_face_index_sets_the_flag_and_draws_nothing_for_it():
    verts, faces, cam = _scene("orbit_550x802")
    W, H = cam.image_width, cam.image_height
    bad = faces.copy()
    bad[100] = [0, 1, len(verts) + 7]
    bad[200] = [-3, 1, 2]
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    gt = _gt(W, H).to(DEV)
    a = mesh_overlay(torch.tensor(verts, device=DEV), torch.tensor(bad, device=DEV), cam, gt, error_flag=flag)
    torch.cuda.synchronize()
    assert int(flag.item()) == 1
    m = mo.Mesh(bad, W, H, verts=verts, block=camera_block(cam).numpy())
    assert not ((m.face_id == 100) | (m.face_id == 200)).any()
    ref = mo.quantize(mo.composite(m.rgba(mo.adjacency_loop(bad)), gt.cpu().numpy(), 0.5))
    assert (a.cpu().numpy() == ref).all()


# ---- GraphedRender(mesh_opacity=...) against eager mesh_overlay over the same float render -------------------------
def test_graphed_render_mesh_overlay_equals_eager_and_never_recaptures():
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _eager, _flame_setup, _rig

    pc = _flame_setup()
    cams = _rig(W_IMG, H_IMG)
    bg = torch.tensor([1.0, 1.0, 1.0])
    F = pc.faces.shape[0]
    colors = torch.rand(F, 3, generator=torch.Generator().manual_seed(7)).to(DEV)
    view = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", warm_cameras=cams, warm_timesteps=range(8),
                         mesh_opacity=0.5, face_colors=colors)
    plain = GraphedRender(pc, W_IMG, H_IMG, bg, outputs="both", warm_cameras=cams, warm_timesteps=range(8))
    checks = [(0, 0, 0.5, None), (1, 3, 0.5, None), (2, 5, 0.8, None), (3, 2, 0.8, torch.rand(F, 3).to(DEV)),
              (0, 6, 0.25, torch.rand(1, F, 3).to(DEV))]
    for ci, t, o, new_colors in checks:
        if new_colors is not None:
            colors = new_colors.reshape(F, 3)
        view.set_inputs(camera=cams[ci], timestep=t, mesh_opacity=o, face_colors=new_colors)
        view.run(check=True)
        plain.set_inputs(camera=cams[ci], timestep=t)
        plain.run(check=True)
        torch.cuda.synchronize()
        ref = _eager(pc, cams[ci], t, bg)
        assert torch.equal(view.image, ref["render"])
        want = mesh_overlay(pc.verts, pc.faces, cams[ci], ref["render"], mesh_opacity=o, face_colors=colors)
        assert torch.equal(view.display, want), f"camera {ci}, timestep {t}, opacity {o}"
        rgba = MeshRenderer().render_from_camera(pc.verts, pc.faces, cams[ci].to(DEV), face_colors=colors)["rgba"]
        off = rgba[0, ..., 3] == 0
        assert off.float().mean() > 0.2 and (~off).float().mean() > 0.02
        assert torch.equal(view.display[off], plain.display[off])
        assert torch.equal(plain.display, ref["display_u8"])
    assert view.captures == 1
    assert int(view.mesh_error.item()) == 0


@pytest.mark.parametrize("name", ["head_gl", "flame_gl_colors"])
def test_shim_reproduces_the_reference_golden(name):
    """tests/golden/mesh_vectors.npz holds the REAL reference renderer's outputs (use_opengl path): the reference's
    call order on the shim reproduces its rast id channel and its rgba."""
    from types import SimpleNamespace

    from tests.test_oracle_mesh_golden import _case, _tol

    verts, faces, c = _case(name)
    W, H, _ = (int(x) for x in c["size"])
    blk = torch.tensor(c["block"])
    cam = SimpleNamespace(world_view_transform=blk[:16].reshape(4, 4).to(DEV),
                          full_proj_transform=blk[16:32].reshape(4, 4).to(DEV), image_width=W, image_height=H)
    fc = None if "face_colors" not in c else torch.tensor(c["face_colors"], device=DEV)[None]
    v = torch.tensor(verts, device=DEV)[None].requires_grad_(True)
    rast, _, _, rgba = _reference_call_order(cam, v, torch.tensor(faces, device=DEV), face_colors=fc)
    assert torch.equal(rast[0, ..., 3].cpu(), torch.tensor(c["rast"][..., 3]))
    assert (rgba[0].cpu() - torch.tensor(c["rgba"])).abs().max() <= _tol(name)
