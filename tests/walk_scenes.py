"""Seeded scenes that drive every branch of the backward blend's walk (blend.cu backward_task), and a host census of
what each warp of that walk does, restated from the oracle's state.

A scene is a row of 16x16 tiles.  Tile t holds L_t faint splats (opacity 0.01 .. 0.05, so no pixel's walk stops on
T < 1e-4) that stay inside the tile (radius <= 5 around a point within 2 px of the tile centre), at distinct depths:
the tile's list is exactly those L_t splats.  A tile with `deep` set puts its deepest splat at the centre with a
footprint that reaches all eight 8x4 blocks, so every warp of the tile walks n = L_t instances; the other tiles end
their warps' walks wherever their last contributing splat lies.  The list lengths are chosen around the 32-entry
chunk edges (n mod 32 in {0, 1, 31}), from one chunk to five (the 3-slot id ring reused), and their sums put the
tiles' first stream positions on every residue mod 16.

Census of one walk (per tile, the backward blend's own schedule):
    K        2 (heavy: list length >> 5 >= max(1, heavy_bwd >> 5), four warps of two bands) or 4 (two warps)
    n        the largest n_contrib over the warp's pixels; chunks = ceil(n / 32)
    visits   stream positions below n whose block-mask byte (the oracle's accepted, live pairs) has one of the warp's
             bits; walked in reverse, chunk c holding reverse indices 32 c .. 32 c + 31, sent three at a time
"""
from __future__ import annotations

import numpy as np
import torch

from tests import adversarial_scenes as A

F32 = np.float32
DEFAULT_HEAVY_BWD = 2048

# (tile list lengths, deep flags) per scene; the last tile of each ends the stream
WALK = {
    "chunk_edges": ([32, 33, 31, 63, 64, 65, 96, 97, 5, 1, 128, 129, 159, 7, 161, 40],
                    [1, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 0, 1, 1]),
    "ragged": ([3, 47, 90, 17, 33, 70, 2, 100, 12, 64, 35, 0, 9, 140, 26, 95],
               [0, 1, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0, 1, 0, 0, 0]),
    "residues": ([33, 49, 33, 17, 49, 33, 49, 81, 33, 49, 33, 33, 49, 1, 33, 49],   # each first position one past
                 [1, 1, 0, 1, 1, 1, 0, 1, 1, 1, 1, 0, 1, 1, 1, 1]),                 # the last mod 16
}


def build(name, seed=0):
    """The scene `name` of WALK: activated CPU tensors as tests/adversarial_scenes.py builds them, one row of tiles."""
    lens, deep = WALK[name]
    W, H = 16 * len(lens), 16
    f = A.default_focal(W, H)
    cam, g = A.camera(W, H, f), torch.Generator().manual_seed(seed)
    us, vs, zs, sig, op = [], [], [], [], []
    for t, (L, d) in enumerate(zip(lens, deep)):
        if L == 0:
            continue
        cx, cy = 16 * t + 7.5, 7.5
        u = cx + A._uniform(g, L, -2.0, 2.0)
        v = cy + A._uniform(g, L, -2.0, 2.0)
        s = A._uniform(g, L, 0.6, 1.3)
        o = A._uniform(g, L, 0.01, 0.05)
        z = 2.0 + 0.01 * t + 2e-4 * torch.randperm(L, generator=g).numpy()
        if d:   # deepest: centred, reaches every block of the tile (alpha ~ 0.3 exp(-4.5^2 / (2 (1.5^2 + 0.3))) > 1/255)
            k = int(np.argmax(z))
            u[k], v[k], s[k], o[k] = cx, cy, 1.5, 0.3
        us.append(u), vs.append(v), zs.append(z), sig.append(s), op.append(o)
    u, v, z, sigma_px, opac = (np.concatenate(a) for a in (us, vs, zs, sig, op))
    P = u.size
    perm = torch.randperm(P, generator=g).numpy()       # a tile's splats are not consecutive ids
    u, v, z, sigma_px, opac = u[perm], v[perm], z[perm], sigma_px[perm], opac[perm]
    xyz = A.unproject(cam, W, H, u, v, z)
    s = sigma_px * z / f
    # largest axis sigma: the radius stays 3 sqrt(sigma^2 + 0.3) <= 5; anisotropic, so the rotation has a gradient
    scales = np.stack([s, 0.8 * s, 0.6 * s], 1)
    sc = A._scene(cam, W, H, xyz, scales, A._rotations(g, P), opac, A._shs(g, P, 0), 0)
    sc["name"] = name
    return sc


def _heavy(length, heavy_bwd):
    """tile_sort.cu: a tile is heavy for the backward from bucket min(62, len >> 5) >= min(62, max(1, heavy_bwd >> 5))."""
    return length > 0 and min(62, length >> 5) >= min(62, max(1, heavy_bwd >> 5))


def block_masks(st):
    """Per stream position, the forward's block-mask byte: bit 2 band + half for each 8x4 block in which the instance
    was accepted by a pixel before that pixel's n_contrib."""
    t = A.pair_table(st)
    took = (t["power"] <= 0) & (t["alpha"] >= A.ALPHA_MIN) & t["live"]
    x, y = t["pix"] % st.W, t["pix"] // st.W
    bit = 2 * ((y % 16) // 4) + (x % 16) // 8
    mask = np.zeros(st.N, np.uint8)
    np.bitwise_or.at(mask, t["j"][took].astype(np.int64), (1 << bit[took]).astype(np.uint8))
    return mask


def census(st, heavy_bwd=DEFAULT_HEAVY_BWD):
    """One record per walking warp (n > 0): tile, K, warp, n, chunks, visits, fill (visits mod 3), straddle (a batch
    of three visits spans two chunks), x16 (range.x mod 16), last (the tile's run ends at the stream's end)."""
    W, H = st.W, st.H
    gx = (W + 15) // 16
    mask = block_masks(st)
    nc = st.n_contrib
    out = []
    for tile in range(st.ranges.shape[0]):
        r0, r1 = int(st.ranges[tile, 0]), int(st.ranges[tile, 1])
        K = 2 if _heavy(r1 - r0, heavy_bwd) else 4
        tx, ty = tile % gx, tile // gx
        for w in range(8 // K):
            half, band0 = w & 1, (w >> 1) * K
            cols = slice(16 * tx + 8 * half, min(16 * tx + 8 * half + 8, W))
            rows = slice(16 * ty + 4 * band0, min(16 * ty + 4 * (band0 + K), H))
            n = int(nc[rows, cols].max()) if nc[rows, cols].size else 0
            if n == 0:
                continue
            bits = sum(1 << (2 * (band0 + i) + half) for i in range(K))
            q = np.arange(n)                                    # reverse index: position n - 1 - q
            vis = q[(mask[r0 + n - 1 - q] & bits) != 0]
            chunk = vis // 32
            batch = np.arange(vis.size) // 3
            straddle = bool(np.any([np.unique(chunk[batch == b]).size > 1 for b in np.unique(batch)]))
            out.append(dict(tile=tile, K=K, warp=w, n=n, chunks=(n + 31) // 32, visits=int(vis.size),
                            fill=int(vis.size % 3), straddle=straddle, x16=r0 % 16, last=r1 == st.N))
    return out


def reached(records):
    """The walk items a census reaches, as (K, item, value) triples."""
    got = set()
    for r in records:
        K = r["K"]
        got |= {(K, "fill", r["fill"]), (K, "n_mod_32", r["n"] % 32), (K, "chunks", min(r["chunks"], 4)),
                (K, "x16", r["x16"])}
        if r["straddle"]:
            got.add((K, "straddle", True))
        if r["last"]:
            got.add((K, "last", True))
    return got


# every item the walk scenes must reach under each K: the end-of-walk batch fill, a batch across a chunk boundary,
# n on and beside the chunk edges, one to four-or-more chunks (the id ring's slots reused), every alignment of the
# mask (mod 16) bulk copies, which covers the id copies' (mod 4), and a tile whose list ends the stream (the reads into the slack)
# ... with the colour backward and with the depth plane (its tenth row, dL/dz, in every batch slot): each scene runs
# in both (tests/test_gpu_backward_walk.py), and RUNS lists the (depth plane, heavy_bwd) runs of those tests
RUNS = [(depth, heavy) for depth in (False, True) for heavy in (DEFAULT_HEAVY_BWD, 32)]
WANTED = {(depth, K, item, v) for depth in (False, True) for K in (2, 4) for item, vals in (
    ("fill", (0, 1, 2)), ("straddle", (True,)), ("n_mod_32", (0, 1, 31)), ("chunks", (1, 2, 3, 4)),
    ("x16", tuple(range(16))), ("last", (True,))) for v in vals}


def bucket(length):
    """tile_sort.cu's length bucket of the heaviest-first order (0: heaviest; empty lists last)."""
    return 63 if length == 0 else 62 - min(62, length >> 5)


def views_interleave(states):
    """The global tile order of a K-view frame (views' tiles concatenated, ordered by bucket) interleaves the views:
    some tile of one view lies strictly between two tiles of another in every order the buckets allow."""
    bk = [np.array([bucket(int(r[1]) - int(r[0])) for r in st.ranges]) for st in states if st is not None]
    for a in range(len(bk)):
        for b in range(len(bk)):
            if a != b and np.any((bk[b] > bk[a].min()) & (bk[b] < bk[a].max())):
                return True
    return False
