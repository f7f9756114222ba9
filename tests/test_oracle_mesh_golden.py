"""CPU: the mesh overlay's numpy restatement composed the way the fused kernels compose it -- per-face shading from the
camera block, antialiasing, row order, and for the reference's CUDA context its //8 render size and bilinear resize --
against tests/golden/mesh_vectors.npz, which the REAL reference mesh renderer produced (tests/golden/make_golden_mesh.py,
nvdiffrast stubbed by the oracle's rasterization in nvdiffrast's layouts)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import mesh_oracle as mo

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["head_gl", "head_cuda_ragged", "flame_gl_colors", "flame_cuda"]


def _tol(name):
    """rgba tolerance.  The reference forms camera-space vertices with a float32 bmm and takes edge differences after
    the translation is added; on the FLAME template's millimetre faces at 0.6 m that rounding alone moves a normal by
    up to 5.5e-6 (the kernels round the same expression in another order), so those cases get 1e-5."""
    return 1e-5 if name.startswith("flame") else 2e-6


def _case(name):
    g = np.load(os.path.join(GOLDEN, "mesh_vectors.npz"))
    if name.startswith("flame"):
        t = np.load(os.path.join(GOLDEN, "flame_template_topology.npz"))
        verts, faces = t["verts"] - t["verts"].mean(0, keepdims=True), t["faces"]
    else:
        verts, faces = g["head/verts"], g["head/faces"]
    c = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    return verts, faces.astype(np.int64), c


def _oracle_rgba(verts, faces, c):
    """The reference's rgba from the oracle: winners of the recorded clip coordinates at the render size, the fused
    route's per-face shading (camera block, OpenGL frame), antialias, flip to row 0 = top, the CUDA context's resize."""
    W, H, gl = (int(x) for x in c["size"])
    w, h = (W, H) if gl else (W // 8 * 8, H // 8 * 8)
    m = mo.Mesh(faces, w, h, pos=c["verts_clip"])
    shade = mo.Mesh(faces, w, h, verts=verts, block=c["block"], face_colors=c.get("face_colors"))
    fid = m.face_id
    rgba = np.empty((h, w, 4), np.float32)
    rgba[..., :3] = np.where(fid[..., None] >= 0, shade.rgb[np.maximum(fid, 0)], np.float32(1))
    rgba[..., 3] = fid >= 0
    out = m.antialias(rgba, mo.adjacency_loop(faces))[::-1]
    if not gl:
        out = F.interpolate(torch.from_numpy(out.copy()).permute(2, 0, 1)[None], (H, W), mode="bilinear")[0]
        out = out.permute(1, 2, 0).numpy()
    return m, shade, fid, np.ascontiguousarray(out)


@pytest.mark.parametrize("name", CASES)
def test_oracle_composes_the_reference_outputs(name):
    verts, faces, c = _case(name)
    m, shade, fid, rgba = _oracle_rgba(verts, faces, c)
    assert (c["rast"][..., 3].astype(np.int64) - 1 == fid).all()
    assert (fid >= 0).sum() > 100
    tol = _tol(name)
    assert np.abs(rgba - c["rgba"]).max() <= tol
    W, H, gl = (int(x) for x in c["size"])
    if gl:   # un-antialiased maps: the per-face diffuse / normal z where covered, the background elsewhere
        f = fid[::-1]
        diffuse = np.where(f[..., None] >= 0, shade.rgb[np.maximum(f, 0)], np.float32(1))
        if "face_colors" not in c:
            assert np.abs(diffuse - c["diffuse"]).max() <= tol
        assert np.abs(np.where(f >= 0, np.clip(c["normal"][..., 2], 0, 1), 1) - c["diffuse"][..., 0]).max() <= tol
    # render.py's composite bytes; a value whose x*255 + 0.5 lies within 1e-4 (or the rgba tolerance's reach) of an
    # integer may round either way
    comp = mo.composite(rgba, c["gt"], 0.5)
    ours = mo.quantize(comp)
    x = np.moveaxis(comp, 0, -1) * 255 + 0.5
    near = np.abs(x - np.round(x)) < max(1e-4, 255 * tol)
    diff = ours.astype(int) - c["composite_u8"].astype(int)
    print(f"{name}: {int(near.sum())} near-tie values, {int((diff != 0).sum())} differ")
    assert (diff[~near] == 0).all() and np.abs(diff).max() <= 1


@pytest.mark.parametrize("name", ["head_gl", "flame_gl_colors"])
def test_fused_route_equals_the_reference_at_native_size(name):
    """The fused kernels' route (clip coordinates from the camera block, row 0 at the top, no flip) against the
    reference's use_opengl output."""
    verts, faces, c = _case(name)
    W, H, _ = (int(x) for x in c["size"])
    m = mo.Mesh(faces, W, H, verts=verts, block=c["block"], face_colors=c.get("face_colors"))
    rgba = m.rgba(mo.adjacency_loop(faces))
    bad = np.abs(rgba - c["rgba"]).max(-1) > _tol(name)
    print(f"{name}: {int(bad.sum())} of {W * H} pixels differ")
    assert not bad.any()
