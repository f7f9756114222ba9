"""CPU: the mesh rasterizer's numpy restatement (tests/mesh_oracle.py) against independent anchors -- a float64 ray cast,
exact single coverage of a tessellated plane, even coverage of a closed mesh, face permutation, near-plane and
guard-band clipping, the analytic antialiasing weight at a boundary edge, and a float64 silhouette classification."""
import math
import os

import numpy as np
import pytest
import torch

from gaussianavatars_b200 import synthetic as syn
from gaussianavatars_b200.graph import camera_block
from gaussianavatars_b200.mesh import mesh_adjacency
from tests import mesh_oracle as mo


def _block(cam):
    return camera_block(cam).numpy()


def _clip64(verts, block):
    v = np.asarray(verts, np.float64)
    M = np.asarray(block, np.float64)[16:32].reshape(4, 4)
    return np.concatenate([v, np.ones((len(v), 1))], 1) @ M


def _ray_cast(clip, faces, W, H):
    """float64: nearest face hit by the ray through every pixel centre (homogeneous barycentric solve, hits inside
    -w <= z <= w), the runner-up's depth, and the distance in pixels to the nearest projected edge of a hit face."""
    cx = (np.arange(W) + 0.5) / (W / 2) - 1
    cy = (np.arange(H) + 0.5) / (H / 2) - 1
    X, Y = np.meshgrid(cx, cy)
    best = np.full((H, W), np.inf)
    second = np.full((H, W), np.inf)
    fid = np.full((H, W), -1)
    edge_d = np.full((H, W), np.inf)
    scr = np.stack([(clip[:, 0] / clip[:, 3] + 1) * W / 2, (clip[:, 1] / clip[:, 3] + 1) * H / 2], 1)
    PX, PY = (np.arange(W) + 0.5)[None, :], (np.arange(H) + 0.5)[:, None]
    for f, (i, j, k) in enumerate(faces):
        v = clip[[i, j, k]]
        a = np.stack([v[:, 0][None, None] - X[..., None] * v[:, 3][None, None],
                      v[:, 1][None, None] - Y[..., None] * v[:, 3][None, None],
                      np.ones((H, W, 3))], -2)
        rhs = np.zeros((H, W, 3))
        rhs[..., 2] = 1
        det = np.linalg.det(a)
        ok = np.abs(det) > 1e-300
        lam = np.zeros((H, W, 3))
        lam[ok] = np.linalg.solve(a[ok], rhs[ok][..., None])[..., 0]
        p = lam @ v
        hit = ok & (lam >= 0).all(-1) & (p[..., 3] > 0) & (p[..., 2] >= -p[..., 3]) & (p[..., 2] <= p[..., 3])
        z = np.where(hit, p[..., 2] / np.where(hit, p[..., 3], 1), np.inf)
        closer = z < best
        second = np.where(closer, best, np.minimum(second, z))
        best = np.where(closer, z, best)
        fid = np.where(closer, f, fid)
        s = scr[[i, j, k]]
        near = np.inf
        for e in range(3):
            a0, a1 = s[e], s[(e + 1) % 3]
            d = a1 - a0
            L = max(np.hypot(*d), 1e-30)
            t = np.clip(((PX - a0[0]) * d[0] + (PY - a0[1]) * d[1]) / (L * L), 0, 1)
            near = np.minimum(near, np.hypot(PX - (a0[0] + t * d[0]), PY - (a0[1] + t * d[1])))
        edge_d = np.minimum(edge_d, np.where(np.isfinite(z) | (near < 2), near, np.inf))
    return fid, best, second, edge_d


def _head(W, H, n_lat=8, n_lon=12, r=1.0, az=20.0, fovy=20.0):
    verts, faces = syn.head_mesh(n_lat=n_lat, n_lon=n_lon)
    cam = syn.orbit_camera(W, H, r=r, fovy_deg=fovy, azimuth_deg=az)
    return np.asarray(verts, np.float32), np.asarray(faces, np.int64), _block(cam)


@pytest.mark.parametrize("W,H,az", [(48, 40, 20.0), (37, 29, -65.0)])
def test_winner_equals_float64_ray_cast_away_from_edges_and_ties(W, H, az):
    verts, faces, blk = _head(W, H, az=az)
    m = mo.Mesh(faces, W, H, verts=verts, block=blk)
    fid, best, second, edge_d = _ray_cast(_clip64(verts, blk), faces, W, H)
    with np.errstate(invalid="ignore"):
        safe = (edge_d > 1.0 / 256) & ~(np.abs(second - best) <= 1e-6 * np.maximum(1.0, np.abs(best)))
    assert safe.mean() > 0.5
    assert (fid >= 0).sum() > 0.2 * W * H
    bad = safe & (m.face_id != fid)
    assert not bad.any(), f"{bad.sum()} pixels differ from the ray cast"


def test_tessellated_plane_on_pixel_centres_is_covered_exactly_once():
    W, H = 20, 16
    g = np.random.default_rng(3)
    cols, rows = np.arange(2, 18), np.arange(1, 15)   # vertices on the centres of these pixels
    gx, gy = np.meshgrid(cols, rows)
    X, Y = gx + 0.5, gy + 0.5
    pos = np.stack([X / (W / 2) - 1, Y / (H / 2) - 1, np.full_like(X, 0.5, dtype=float), np.ones_like(X, float)],
                   -1).reshape(-1, 4).astype(np.float32)
    nc = len(cols)
    tris = []
    for r in range(len(rows) - 1):
        for c in range(nc - 1):
            a, b, d, e = r * nc + c, r * nc + c + 1, (r + 1) * nc + c, (r + 1) * nc + c + 1
            if g.random() < 0.5:
                tris += [(a, b, e), (a, e, d)]
            else:
                tris += [(a, b, d), (b, e, d)]
            if g.random() < 0.5:
                tris[-1] = tris[-1][::-1]
    m = mo.Mesh(np.array(tris), W, H, pos=pos)
    assert m.coverage.max() == 1
    inner = m.coverage[rows[0] + 1:rows[-1], cols[0] + 1:cols[-1]]
    assert (inner == 1).all()


def test_closed_mesh_is_covered_an_even_number_of_times():
    W, H = 41, 33
    verts, faces, blk = _head(W, H, n_lat=9, n_lon=14, az=33.0)
    m = mo.Mesh(faces, W, H, verts=verts, block=blk)
    assert (m.coverage > 0).sum() > 0.2 * W * H
    assert (m.coverage % 2 == 0).all()


def test_permuting_faces_permutes_ids():
    W, H = 40, 32
    verts, faces, blk = _head(W, H)
    perm = np.random.default_rng(0).permutation(len(faces))
    a = mo.Mesh(faces, W, H, verts=verts, block=blk).face_id
    b = mo.Mesh(faces[perm], W, H, verts=verts, block=blk).face_id
    assert ((a >= 0) == (b >= 0)).all()
    assert (a[a >= 0] == perm[b[b >= 0]]).all()


def test_near_plane_and_guard_band_clipping_match_the_ray_cast():
    W, H = 32, 24
    cam = syn.look_at_camera(W, H, 60.0, 48.0, znear=0.01, zfar=100.0)   # the reference's projection: z in [0, w]
    blk = _block(cam)
    znear_eff = 100.0 * 0.01 / (2 * 100.0 - 0.01)                       # -w <= z: view depth >= ~0.005
    tx, ty = math.tan(math.radians(30)), math.tan(math.radians(24))
    verts = np.array([
        # straddles the effective near plane
        [-0.5 * tx * 0.004, -0.5 * ty * 0.004, 0.004], [0.5 * tx * 0.02, -0.3 * ty * 0.02, 0.02],
        [0.0, 0.6 * ty * 0.006, 0.006],
        # one vertex ~1e6 px off screen
        [-0.3 * tx, 0.2 * ty, 1.0], [0.2 * tx, 0.5 * ty, 1.0], [1e6 / (W / 2) * tx * 2.0, 0.0, 2.0],
    ], np.float32)
    faces = np.array([[0, 1, 2], [3, 4, 5]])
    m = mo.Mesh(faces, W, H, verts=verts, block=blk)
    assert m.inside[0] != 7 and m.inside[1] != 7           # both faces are clipped
    assert min(verts[:3, 2]) < znear_eff < max(verts[:3, 2])
    fid, best, second, edge_d = _ray_cast(_clip64(verts, blk), faces, W, H)
    safe = edge_d > 1.0 / 256
    assert (fid[safe] == 0).any() and (fid[safe] == 1).any()
    assert (m.face_id[safe] == fid[safe]).all()


@pytest.mark.parametrize("delta", [0.0625, 0.25, 0.4375, 0.75, 0.9375])
def test_boundary_edge_blend_weight_is_the_analytic_coverage(delta):
    W, H, c = 16, 12, 7
    X0 = c + 0.5 + delta
    pts = np.array([[X0, -100.0], [X0, 200.0], [-300.0, 50.0]])
    pos = np.stack([pts[:, 0] / (W / 2) - 1, pts[:, 1] / (H / 2) - 1, np.zeros(3), np.ones(3)], 1).astype(np.float32)
    faces = np.array([[0, 1, 2]])
    m = mo.Mesh(faces, W, H, pos=pos)
    adj = mesh_adjacency(torch.tensor(faces)).numpy()
    assert (adj == -1).all()
    alpha = m.antialias(m.colors(), adj)[..., 3]
    if delta < 0.5:
        assert (alpha[:, c] == np.float32(0.5 + delta)).all()
        assert (alpha[:, c + 1] == 0).all()
    else:
        assert (alpha[:, c] == 1).all()
        assert (alpha[:, c + 1] == np.float32(delta - 0.5)).all()
    assert (alpha[:, :c] == 1).all() and (alpha[:, c + 2:] == 0).all()


def _flame_template():
    t = np.load(os.path.join(os.path.dirname(__file__), "golden", "flame_template_topology.npz"))
    v = t["verts"]
    return v - v.mean(0, keepdims=True), t["faces"].astype(np.int64)


def test_flame_template_topology_fixture():
    verts, faces = _flame_template()
    adj = mesh_adjacency(torch.tensor(faces)).numpy()
    assert verts.shape == (5023, 3) and faces.shape == (9976, 3)
    assert (adj == -1).sum() == 62 and (adj >= 0).sum() == 2 * 14_933
    assert (adj == mo.adjacency_loop(faces)).all()


@pytest.mark.parametrize("mesh", ["head", "flame_template"])
def test_silhouette_classification_matches_float64(mesh):
    W, H = 64, 48
    if mesh == "head":
        verts, faces, blk = _head(W, H, n_lat=12, n_lon=20, az=50.0)
    else:
        verts, faces = _flame_template()
        blk = _block(syn.orbit_camera(W, H, r=0.6, fovy_deg=20.0, azimuth_deg=50.0, elevation_deg=10.0))
    adj = mesh_adjacency(torch.tensor(faces)).numpy()
    m = mo.Mesh(faces, W, H, verts=verts, block=blk)
    sil = m.silhouette(adj)
    clip = _clip64(verts, blk)
    s = np.stack([(clip[:, 0] / clip[:, 3] + 1) * W / 2, (clip[:, 1] / clip[:, 3] + 1) * H / 2], 1)

    def orient(a, b, p):
        return (b[..., 0] - a[..., 0]) * (p[..., 1] - a[..., 1]) - (b[..., 1] - a[..., 1]) * (p[..., 0] - a[..., 0])

    n_checked = n_boundary = 0
    for f in range(len(faces)):
        for k in range(3):
            a, b, o = faces[f, k], faces[f, (k + 1) % 3], faces[f, (k + 2) % 3]
            so = orient(s[a], s[b], s[o])
            n = adj[f, k]
            if n < 0:
                if abs(so) >= 1e-2:
                    assert sil[f, k], (f, k)
                    n_boundary += 1
                continue
            u = [j for j in faces[n] if j not in (a, b)][0]
            su = orient(s[a], s[b], s[u])
            if min(abs(so), abs(su)) < 1e-2:
                continue
            assert sil[f, k] == (so * su > 0), (f, k)
            n_checked += 1
    assert n_checked > 0.9 * 3 * len(faces) - 62
    assert 0 < sil.sum() < 0.5 * sil.size
    assert n_boundary == (62 if mesh == "flame_template" else 0)


def test_adjacency_builder_matches_a_python_loop():
    verts, faces = syn.head_mesh(n_lat=7, n_lon=9)
    faces = np.asarray(faces)
    # open it (drop faces) and add a non-manifold fin: three faces on one edge -> boundary for all three
    f = np.concatenate([faces[5:], [[faces[10, 0], faces[10, 1], 0]]])
    got = mesh_adjacency(torch.tensor(f)).numpy()
    assert (got == mo.adjacency_loop(f)).all()
    assert (got == -1).sum() > 3
