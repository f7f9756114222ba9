"""Generates two fixtures for the mesh overlay (csrc/mesh.cu), from the reference checkout (/root/reference, read-only):

  flame_template_topology.npz  the FLAME template mesh (flame_model/assets/flame/head_template_mesh.obj) as verts
                               (5023,3) float32 and faces (9976,3) int32: real topology with boundary edges (neck,
                               eye sockets) for the silhouette tests.
  mesh_vectors.npz             the REAL reference mesh renderer (mesh_renderer/__init__.py NVDiffRenderer) run on the
                               CPU with `nvdiffrast.torch` stubbed by the numpy oracle (tests/mesh_oracle.py) in
                               nvdiffrast's layouts, `Tensor.cuda` and `device="cuda"` mapped to the CPU.  Per case it
                               records the verts_clip the reference hands to rasterize, the rast it got back, the
                               returned {rgba, normal, diffuse, albedo} and render.py's composite bytes over a random
                               ground truth (render.py:75-81).  That pins everything the reference does AROUND the
                               rasterizer -- the view / projection negations and transposes, the flips, normals,
                               lighting, the face-colour gather, the background, the CUDA context's //8 size and
                               bilinear resize, the composite -- to its real code; the rasterization itself is
                               anchored independently (tests/test_oracle_mesh.py).

    python tests/golden/make_golden_mesh.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
from tests import mesh_oracle as mo  # noqa: E402
from tests import ref_import  # noqa: E402
from gaussianavatars_b200 import synthetic as syn  # noqa: E402
from gaussianavatars_b200.graph import camera_block  # noqa: E402

OBJ = os.path.join(ref_import.REF, "flame_model", "assets", "flame", "head_template_mesh.obj")


def flame_template():
    verts, faces = [], []
    with open(OBJ) as f:
        for line in f:
            if line.startswith("v "):
                verts.append([float(x) for x in line.split()[1:4]])
            elif line.startswith("f "):
                faces.append([int(t.split("/")[0]) - 1 for t in line.split()[1:4]])
    return np.asarray(verts, np.float32), np.asarray(faces, np.int32)


_calls = {}


def _rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    h, w = int(resolution[0]), int(resolution[1])
    p = pos[0].detach().numpy().astype(np.float32)
    m = mo.Mesh(tri.numpy(), w, h, pos=p)
    rast = np.zeros((1, h, w, 4), np.float32)
    fid = m.face_id
    key = (m.winner >> np.uint64(32)).astype(np.uint32)
    zbits = np.where(key & np.uint32(0x80000000), key & np.uint32(0x7FFFFFFF), ~key).astype(np.uint32)
    rast[0, ..., 2] = np.where(fid >= 0, zbits.view(np.float32), 0)
    rast[0, ..., 3] = fid + 1
    _calls["verts_clip"], _calls["rast"] = p, rast[0]
    return torch.from_numpy(rast), torch.zeros(1, h, w, 4)


def _antialias(color, rast, pos, tri, topology_hash=None, pos_gradient_boost=1.0):
    h, w = color.shape[1:3]
    m = mo.Mesh(tri.numpy(), w, h, pos=pos[0].detach().numpy().astype(np.float32))
    return torch.from_numpy(m.antialias(color[0].detach().numpy(), mo.adjacency_loop(tri.numpy()))[None])


def reference_renderer(use_opengl):
    ref_import.prepare()
    dr = sys.modules["nvdiffrast.torch"]
    sys.modules["nvdiffrast"].torch = dr
    dr.RasterizeCudaContext = dr.RasterizeGLContext = lambda *a, **k: types.SimpleNamespace()
    dr.rasterize, dr.antialias = _rasterize, _antialias
    torch.Tensor.cuda = lambda self, *a, **k: self
    real_tensor = torch.tensor

    def tensor_cpu(*a, **k):
        k.pop("device", None)
        return real_tensor(*a, **k)

    torch.tensor = tensor_cpu
    from mesh_renderer import NVDiffRenderer  # noqa: E402  (REAL reference code)

    return NVDiffRenderer(use_opengl=use_opengl)


CASES = {   # name: (mesh, W, H, use_opengl, face colours, camera)
    # flame: the template centred at its float32 mean (tests/test_oracle_mesh_golden.py rebuilds it from the fixture)
    "head_gl": ("head", 48, 40, True, False, dict(r=1.0, az=25.0, el=5.0)),
    "head_cuda_ragged": ("head", 43, 29, False, True, dict(r=1.0, az=-30.0, el=-8.0)),
    "flame_gl_colors": ("flame", 40, 48, True, True, dict(r=0.6, az=35.0, el=10.0)),
    "flame_cuda": ("flame", 48, 40, False, False, dict(r=0.6, az=-60.0, el=0.0)),
}


def main():
    fv, ff = flame_template()
    np.savez_compressed(os.path.join(HERE, "flame_template_topology.npz"), verts=fv, faces=ff)
    hv, hf = syn.head_mesh(n_lat=7, n_lon=10)
    meshes = {"head": (np.asarray(hv, np.float32), np.asarray(hf, np.int32)),
              "flame": (fv - fv.mean(0, keepdims=True), ff)}
    out = {}
    g = np.random.default_rng(0)
    for name, (mesh, W, H, gl, colors, c) in CASES.items():
        verts, faces = meshes[mesh]
        cam = syn.orbit_camera(W, H, r=c["r"], fovy_deg=20.0, azimuth_deg=c["az"], elevation_deg=c["el"])
        fc = g.random((1, len(faces), 3)).astype(np.float32) if colors else None
        rnd = reference_renderer(gl)
        with torch.no_grad():
            d = rnd.render_from_camera(torch.from_numpy(verts)[None], torch.from_numpy(faces), cam,
                                       face_colors=None if fc is None else torch.from_numpy(fc))
            gt = torch.from_numpy(g.integers(0, 256, (3, H, W), dtype=np.uint8))
            # render.py:75-81 and its PNG quantisation
            rgba_mesh = d["rgba"].squeeze(0).permute(2, 0, 1)
            rgb_mesh, alpha_mesh = rgba_mesh[:3, :, :], rgba_mesh[3:, :, :]
            mesh_opacity = 0.5
            gtf = gt.float() / 255.0
            rendering_mesh = rgb_mesh * alpha_mesh * mesh_opacity + gtf.to(rgb_mesh) * (
                alpha_mesh * (1 - mesh_opacity) + (1 - alpha_mesh))
            u8 = rendering_mesh.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)
        pre = name + "/"
        out.update({pre + "block": camera_block(cam).numpy(),
                    pre + "size": np.array([W, H, int(gl)]), pre + "verts_clip": _calls["verts_clip"],
                    pre + "rast": _calls["rast"], pre + "gt": gt.numpy(), pre + "composite_u8": u8.numpy()})
        if fc is not None:
            out[pre + "face_colors"] = fc[0]
        for k in ("rgba", "normal", "diffuse", "albedo"):
            out[pre + k] = d[k][0].numpy()
        print(name, {k: tuple(d[k].shape) for k in d}, "covered", int((_calls["rast"][..., 3] > 0).sum()))
    out.update({"head/verts": meshes["head"][0], "head/faces": meshes["head"][1]})   # flame: the topology fixture
    np.savez_compressed(os.path.join(HERE, "mesh_vectors.npz"), **out)


if __name__ == "__main__":
    main()
