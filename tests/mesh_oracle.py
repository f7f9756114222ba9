"""numpy restatement of csrc/mesh.cu (include/gab200_rasterizer.h, gab200_mesh_render): float32 clip coordinates,
clipping and snapping in the kernel's operation order, int64 edge functions with the same fill rule, the same depth keys
and tie rule, the silhouette antialiasing, the flat shading and render.py's composite.  Every float32 operation is
rounded on its own, as the kernel (built with --fmad=false) rounds it, so winner maps, rgba and composite bytes are
expected to agree bit for bit.  Test infrastructure only: the library never imports it."""
import numpy as np

f32 = np.float32
MAXP = 9
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def to_f32(e):
    """int64 -> float32, correctly rounded (|e| < 2^53, so the float64 step is exact)."""
    return np.asarray(e, dtype=np.int64).astype(np.float64).astype(np.float32)


def depth_key(z):
    u = np.asarray(z, dtype=np.float32).view(np.uint32).astype(np.uint64)
    neg = (u & np.uint64(0x80000000)) != 0
    return np.where(neg, (~u) & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))


def clip_coords(verts, block):
    """[v,1] . full_proj (row-vector layout; the 16 floats at block[16:32]), summed left to right."""
    v = np.asarray(verts, dtype=f32)
    M = np.asarray(block, dtype=f32)[16:32].reshape(4, 4)
    return np.stack([((v[:, 0] * M[0, j] + v[:, 1] * M[1, j]) + v[:, 2] * M[2, j]) + M[3, j] for j in range(4)], 1)


def plane_dist(p, k, gx, gy):
    x, y, z, w = p[..., 0], p[..., 1], p[..., 2], p[..., 3]
    return [w + z, w - z, gx * w + x, gx * w - x, gy * w + y, gy * w - y][k]


def inside_all(p, gx, gy):
    ok = p[..., 3] > 0
    for k in range(6):
        ok = ok & (plane_dist(p, k, gx, gy) >= 0)
    return ok


def snap(p, W, H):
    X = (p[..., 0] / p[..., 3] + f32(1)) * f32(0.5 * W)
    Y = (p[..., 1] / p[..., 3] + f32(1)) * f32(0.5 * H)
    return np.rint(X * f32(256)).astype(np.int64), np.rint(Y * f32(256)).astype(np.int64)


def edge_fn(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def owned(dx, dy):
    return (dy < 0) | ((dy == 0) & (dx > 0))


def clip_polygon(P, gx, gy):
    """Sutherland-Hodgman of the rows (x, y, z, w, b0, b1) against the six planes, in the kernel's order."""
    src = [np.asarray(r, dtype=f32) for r in P]
    for k in range(6):
        if not src:
            break
        dst = []
        n = len(src)
        for i in range(n):
            c, d = src[i], src[(i + 1) % n]
            dc, dd = plane_dist(c, k, gx, gy), plane_dist(d, k, gx, gy)
            if dc >= 0:
                dst.append(c)
            if (dc >= 0) != (dd >= 0) and len(dst) < MAXP:
                t = dc / (dc - dd)
                dst.append(c + t * (d - c))
        src = dst
    return src


class Mesh:
    """Setup + raster of one frame.  pos: (V,4) clip coordinates, or verts (V,3) with a camera block."""

    def __init__(self, faces, W, H, verts=None, block=None, pos=None, face_colors=None, background=(1, 1, 1),
                 lighting="front"):
        self.W, self.H = W, H
        self.faces = np.asarray(faces, dtype=np.int64)
        F = self.faces.shape[0]
        self.F = F
        clip = np.asarray(pos, dtype=f32) if pos is not None else clip_coords(verts, block)
        V = clip.shape[0]
        self.gx, self.gy = f32(65536.0) / f32(W), f32(65536.0) / f32(H)
        gx, gy = self.gx, self.gy
        vin = inside_all(clip, gx, gy)
        with np.errstate(all="ignore"):
            sx, sy = snap(clip, W, H)
        self.clip, self.vin, self.sx, self.sy = clip, vin, sx, sy
        bad = ((self.faces < 0) | (self.faces >= V)).any(1)
        self.bad_face = bad
        fi = np.where(bad[:, None], 0, self.faces)
        self.inside = np.where(bad, 0, vin[fi[:, 0]] * 1 + vin[fi[:, 1]] * 2 + vin[fi[:, 2]] * 4)
        self.evx = np.where((self.inside[:, None] >> np.arange(3)) & 1, sx[fi], 0)
        self.evy = np.where((self.inside[:, None] >> np.arange(3)) & 1, sy[fi], 0)
        s = edge_fn(self.evx[:, 0], self.evy[:, 0], self.evx[:, 1], self.evy[:, 1], self.evx[:, 2], self.evy[:, 2])
        self.orient = np.where(self.inside == 7, np.sign(s), 0)
        # polygons
        self.polys = []
        for f in range(F):
            if bad[f]:
                self.polys.append(None)
                continue
            if self.inside[f] == 7:
                idx = fi[f]
                poly = dict(sx=sx[idx], sy=sy[idx], zw=clip[idx, 2] / clip[idx, 3],
                            b0=np.array([1, 0, 0], f32), b1=np.array([0, 1, 0], f32), iw=f32(1) / clip[idx, 3])
            else:
                rows = [np.concatenate([clip[fi[f, k]], [f32(k == 0), f32(k == 1)]]).astype(f32) for k in range(3)]
                pts = clip_polygon(rows, gx, gy)
                if len(pts) < 3 or any(p[3] <= 0 for p in pts):
                    self.polys.append(None)
                    continue
                pts = np.stack(pts)
                px_, py_ = snap(pts, W, H)
                poly = dict(sx=px_, sy=py_, zw=pts[:, 2] / pts[:, 3], b0=pts[:, 4], b1=pts[:, 5], iw=f32(1) / pts[:, 3])
            self.polys.append(poly)
        # flat colours
        self.rgb = np.ones((F, 3), f32)
        if pos is None:
            Wv = np.asarray(block, dtype=f32)[:16].reshape(4, 4)
            v = np.asarray(verts, dtype=f32)
            cam = np.stack([((v[:, 0] * Wv[0, j] + v[:, 1] * Wv[1, j]) + v[:, 2] * Wv[2, j]) + Wv[3, j]
                            for j in range(3)], 1)
            cam[:, 1:] = -cam[:, 1:]
            c = cam[fi]
            e1, e2 = c[:, 1] - c[:, 0], c[:, 2] - c[:, 0]
            nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
            ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
            nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
            ln = np.sqrt(np.maximum((nx * nx + ny * ny) + nz * nz, f32(1e-20)))
            diffuse = np.minimum(np.maximum(nz / ln, f32(0)), f32(1)) if lighting == "front" else np.ones(F, f32)
            albedo = np.ones((F, 3), f32) if face_colors is None else np.asarray(face_colors, f32).reshape(F, 3)
            self.rgb = np.where(bad[:, None], f32(1), albedo * diffuse[:, None]).astype(f32)
        self.background = np.asarray(background, f32)
        self.coverage = np.zeros((H, W), np.int64)
        self.winner = self._raster()

    def _subtris(self, P):
        n = len(P["sx"])
        for j in range(1, n - 1):
            ia, ib, ic = 0, j, j + 1
            ax, ay, bx, by, cx, cy = P["sx"][ia], P["sy"][ia], P["sx"][ib], P["sy"][ib], P["sx"][ic], P["sy"][ic]
            area = edge_fn(ax, ay, bx, by, cx, cy)
            if area == 0:
                continue
            if area < 0:
                bx, by, cx, cy, ib, ic, area = cx, cy, bx, by, ic, ib, -area
            yield (int(ax), int(ay), int(bx), int(by), int(cx), int(cy), ia, ib, ic, int(area))

    def _raster(self):
        W, H = self.W, self.H
        win = np.full((H, W), EMPTY, dtype=np.uint64)
        for f, P in enumerate(self.polys):
            if P is None:
                continue
            xmin, xmax, ymin, ymax = int(P["sx"].min()), int(P["sx"].max()), int(P["sy"].min()), int(P["sy"].max())
            c0, c1 = max(-((128 - xmin) >> 8), 0), min((xmax - 128) >> 8, W - 1)
            r0, r1 = max(-((128 - ymin) >> 8), 0), min((ymax - 128) >> 8, H - 1)
            if c1 < c0 or r1 < r0:
                continue
            px = (256 * np.arange(c0, c1 + 1, dtype=np.int64) + 128)[None, :]
            py = (256 * np.arange(r0, r1 + 1, dtype=np.int64) + 128)[:, None]
            best = np.full((r1 - r0 + 1, c1 - c0 + 1), EMPTY, dtype=np.uint64)
            for (ax, ay, bx, by, cx, cy, ia, ib, ic, area) in self._subtris(P):
                e0, e1, e2 = edge_fn(bx, by, cx, cy, px, py), edge_fn(cx, cy, ax, ay, px, py), edge_fn(ax, ay, bx, by, px, py)
                cov = (((e0 > 0) | ((e0 == 0) & owned(cx - bx, cy - by))) &
                       ((e1 > 0) | ((e1 == 0) & owned(ax - cx, ay - cy))) &
                       ((e2 > 0) | ((e2 == 0) & owned(bx - ax, by - ay))))
                if not cov.any():
                    continue
                self.coverage[r0:r1 + 1, c0:c1 + 1] += cov
                s = (to_f32(e0) * P["zw"][ia] + to_f32(e1) * P["zw"][ib]) + to_f32(e2) * P["zw"][ic]
                z = s / to_f32(area)
                key = (depth_key(z) << np.uint64(32)) | np.uint64(f)
                best = np.where(cov, np.minimum(best, key), best)
            sl = win[r0:r1 + 1, c0:c1 + 1]
            win[r0:r1 + 1, c0:c1 + 1] = np.minimum(sl, best)
        return win

    @property
    def face_id(self):
        """(H,W) int64: winning face index, -1 for background."""
        return np.where(self.winner == EMPTY, -1, (self.winner & np.uint64(0xFFFFFFFF)).astype(np.int64))

    def silhouette(self, adjacency):
        """(F,3) bool: edge k of face f is a silhouette candidate (kernel: silhouette_edge)."""
        F = self.F
        adj = np.asarray(adjacency, np.int64)
        sil = np.zeros((F, 3), bool)
        for k in range(3):
            k1 = (k + 1) % 3
            ok = ((self.inside >> k) & 1).astype(bool) & ((self.inside >> k1) & 1).astype(bool) & (self.orient != 0)
            N = adj[:, k]
            sil[:, k] = ok & (N == -1)
            cand = ok & (N >= 0) & (N < F)
            for f in np.nonzero(cand)[0]:
                n = N[f]
                if self.bad_face[f] or self.bad_face[n]:
                    continue
                ia, ib = self.faces[f, k], self.faces[f, k1]
                others = [j for j in self.faces[n] if j != ia and j != ib]
                if not others:
                    continue
                u = others[0]
                if not self.vin[u]:
                    continue
                s = edge_fn(self.evx[f, k], self.evy[f, k], self.evx[f, k1], self.evy[f, k1], self.sx[u], self.sy[u])
                sil[f, k] = (s > 0 and self.orient[f] > 0) or (s < 0 and self.orient[f] < 0)
        return sil

    def pair_weights(self, adjacency):
        """Antialiasing weights: (wL, wR, wU, wD), each (H,W) float32 -- how far the pixel moves toward that neighbour."""
        H, W = self.H, self.W
        sil = self.silhouette(adjacency)
        out = [np.zeros((H, W), f32) for _ in range(4)]
        for horizontal in (True, False):
            if horizontal:
                kq, kn = self.winner[:, :-1], self.winner[:, 1:]
                rq, cq = np.mgrid[0:H, 0:W - 1]
                rn, cn = rq, cq + 1
            else:
                kq, kn = self.winner[:-1, :], self.winner[1:, :]
                rq, cq = np.mgrid[0:H - 1, 0:W]
                rn, cn = rq + 1, cq
            m = kq != kn
            kq, kn, rq, cq, rn, cn = kq[m], kn[m], rq[m], cq[m], rn[m], cn[m]
            q_occ = kq < kn
            T = (np.where(q_occ, kq, kn) & np.uint64(0xFFFFFFFF)).astype(np.int64)
            ac, ar = np.where(q_occ, cq, cn), np.where(q_occ, rq, rn)
            bc, br = np.where(q_occ, cn, cq), np.where(q_occ, rn, rq)
            ax, ay, bx, by = 256 * ac + 128, 256 * ar + 128, 256 * bc + 128, 256 * br + 128
            tbest = np.full(T.shape, f32(2))
            for k in range(3):
                k1 = (k + 1) % 3
                x0, y0, x1, y1 = self.evx[T, k], self.evy[T, k], self.evx[T, k1], self.evy[T, k1]
                dx, dy = x1 - x0, y1 - y0
                ok = ((np.abs(dx) <= np.abs(dy)) == horizontal) & sil[T, k]
                ea, eb = edge_fn(x0, y0, x1, y1, ax, ay), edge_fn(x0, y0, x1, y1, bx, by)
                ok &= ea != eb
                with np.errstate(all="ignore"):
                    t = to_f32(ea) / to_f32(np.where(ea == eb, 1, ea - eb))
                ok &= (t >= 0) & (t <= 1)
                if horizontal:
                    ok &= (ay >= np.minimum(y0, y1)) & (ay <= np.maximum(y0, y1))
                else:
                    ok &= (ax >= np.minimum(x0, x1)) & (ax <= np.maximum(x0, x1))
                tbest = np.where(ok & (t < tbest), t, tbest)
            has = tbest <= 1
            wa = np.where(has & (tbest < 0.5), f32(0.5) - tbest, f32(0))   # the occluder moves
            wb = np.where(has & (tbest > 0.5), tbest - f32(0.5), f32(0))   # the other pixel moves
            wq = np.where(q_occ, wa, wb).astype(f32)
            wn = np.where(q_occ, wb, wa).astype(f32)
            # q's neighbour n is to the right/below: q's slot R/D, n's slot L/U
            sq, sn = (1, 0) if horizontal else (3, 2)
            out[sq][rq, cq] = wq
            out[sn][rn, cn] = wn
        return out

    def colors(self):
        """(H,W,4) float32 un-antialiased rgba."""
        fid = self.face_id
        rgba = np.empty((self.H, self.W, 4), f32)
        rgba[..., :3] = np.where(fid[..., None] >= 0, self.rgb[np.maximum(fid, 0)], self.background)
        rgba[..., 3] = (fid >= 0).astype(f32)
        return rgba

    def antialias(self, color, adjacency):
        """(H,W,C) float32 -> antialiased, deltas added in the order left, right, up, down."""
        c = np.asarray(color, f32)
        w = self.pair_weights(adjacency)
        H, W = self.H, self.W
        acc = c.copy()
        nb = [(0, -1), (0, 1), (-1, 0), (1, 0)]
        for j, (dr, dc) in enumerate(nb):
            cn = np.empty_like(c)
            rr = np.clip(np.arange(H) + dr, 0, H - 1)
            cc = np.clip(np.arange(W) + dc, 0, W - 1)
            cn[:] = c[rr][:, cc]
            wj = w[j][..., None]
            acc = np.where(wj != 0, acc + wj * (cn - c), acc).astype(f32)
        return acc

    def rgba(self, adjacency=None, antialias=True):
        c = self.colors()
        return self.antialias(c, adjacency) if antialias else c


def composite(rgba, base, opacity):
    """render.py's rgb * a * o + base * (a * (1 - o) + (1 - a)) in float32, (3,H,W); base float (3,H,W) or uint8."""
    o, omo = f32(opacity), f32(1.0 - float(opacity))
    b = np.asarray(base)
    b = b.astype(f32) / f32(255) if b.dtype == np.uint8 else b.astype(f32)
    rgb = np.moveaxis(rgba[..., :3], -1, 0)
    a = rgba[..., 3][None]
    keep = a * omo + (f32(1) - a)
    return (rgb * a) * o + b * keep


def quantize(img_chw):
    """render.py's mul(255).add_(0.5).clamp_(0, 255) -> uint8 (truncation), as (H,W,3)."""
    q = np.clip(np.asarray(img_chw, f32) * f32(255) + f32(0.5), f32(0), f32(255)).astype(np.uint8)
    return np.ascontiguousarray(np.moveaxis(q, 0, -1))


def adjacency_loop(faces):
    """Python-loop restatement of mesh.mesh_adjacency (the test anchor)."""
    faces = np.asarray(faces, np.int64)
    owners = {}
    for f, tri in enumerate(faces):
        for k in range(3):
            a, b = int(tri[k]), int(tri[(k + 1) % 3])
            owners.setdefault((min(a, b), max(a, b)), []).append((f, k))
    adj = np.full(faces.shape, -1, np.int32)
    for lst in owners.values():
        if len(lst) == 2:
            (f0, k0), (f1, k1) = lst
            adj[f0, k0], adj[f1, k1] = f1, f0
    return adj
