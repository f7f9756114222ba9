// mesh.cu -- the tracked mesh drawn over an image: a watertight triangle rasterizer with silhouette antialiasing.
// Replaces what the reference's mesh_renderer (mesh_renderer/__init__.py:183-274) asks of nvdiffrast
// (dr.rasterize + dr.antialias) and, fused, render.py's mesh composite (render.py:75-81).
//
// Compiled with --fmad=false: every float below is rounded op by op in the order written, so the numpy restatement in
// tests/mesh_oracle.py reproduces the snapped vertices, the depth keys and therefore the winner map bit for bit.
//
// Every launch carries a view index: one call draws one vertex set under K cameras (gab200_mesh_render_views), each
// (view, face) projected through row k of a [K,37] camera table into its own face records and its own winner map, and
// view k's pixels read base plane k and write output plane k.  The single-view call is K = 1 of the same kernels, and
// view k of a K-view call is bit for bit the single-view call with camera k and base k: no value crosses views, and
// the only shared step -- the persistent raster warps' division of the work items -- ends in an order-free atomicMin.
//
// Launches (all stream-ordered, no host wait, capturable):
//   mesh_setup_kernel    one thread per (view, face): clip coordinates ([v,1] . full_proj, or given), clip against the
//                        clip volume -w <= z <= w and a guard band of 2^15 px, snap to 1/256 px, flat colour, pixel
//                        bounding box and its number of 8x4 pixel tiles
//   cub InclusiveSum     tiles per (view, face) -> offsets (u64)
//   mesh_silhouette_kernel  (antialias only) one thread per (view, face): which of its edges are screen-space silhouettes
//   mesh_raster_kernel   persistent warps, each an equal share of the (view, face, 8x4 tile) work items of all views
//                        (a face covering 1e5 px is spread over many warps): int64 edge functions with a
//                        top-left rule, z/w at the pixel centre, 64-bit atomicMin of (depth key << 32 | face id)
//   mesh_resolve_kernel  one thread per (view, pixel): shading, silhouette antialiasing from the winners of the pixel and its
//                        4 neighbours, then the requested outputs
// Pixel convention: column c / row r has its centre at (c + 1/2, r + 1/2) with X = (x/w + 1) W/2, Y = (y/w + 1) H/2,
// so row 0 is clip y = -1: the top row of the splat image for a camera's own full_proj_transform, and nvdiffrast's
// row 0 for the reference's y-negated clip coordinates.
#include <cub/cub.cuh>

#include "common.cuh"
#include "kernels.cuh"

namespace gab {
namespace {

constexpr int MAXP = 9;                 // a triangle clipped by 6 planes has at most 9 vertices
constexpr uint64_t EMPTY = ~0ull;       // winner of an uncovered pixel (background)

struct __align__(16) FacePoly {         // clipped polygon of one face, fan from vertex 0
  int n;                                // vertices (0: nothing to draw)
  int c0, r0, c1, r1;                   // covered pixel centres lie in [c0, c1] x [r0, r1]
  int sx[MAXP], sy[MAXP];               // snapped to 1/256 px
  float zw[MAXP];                       // z / w
  float b0[MAXP], b1[MAXP], iw[MAXP];   // barycentrics of the original triangle's vertices 0, 1 and 1 / w
};

struct __align__(16) FaceEdges {        // the unclipped triangle, for the silhouette test of the resolve
  int vx[3], vy[3];
  int inside;                           // bit k: vertex k lies inside the clip volume and the guard band;
                                        // bit 3 + k: edge k is a silhouette (mesh_silhouette_kernel)
  int orient;                           // sign of the snapped triangle's signed area (0 if a vertex is outside)
};

struct MeshParams {
  int V, F, W, H, pos_kind;
  int K;                                // views: the records of view k are [k F, k F + F), its winners [k H W, ...)
  const float* verts;
  const int32_t* faces;
  const int32_t* adj;
  const float* cam;                     // camera block of view 0; view k's at cam + k * GAB200_CAMERA_FLOATS
  float gx, gy;                         // guard band in NDC units: 2^16 / W, 2^16 / H
};

struct PV { float x, y, z, w, b0, b1; };

__device__ __forceinline__ float plane_dist(const PV& v, int k, float gx, float gy) {
  switch (k) {
    case 0: return __fadd_rn(v.w, v.z);
    case 1: return __fsub_rn(v.w, v.z);
    case 2: return __fadd_rn(__fmul_rn(gx, v.w), v.x);
    case 3: return __fsub_rn(__fmul_rn(gx, v.w), v.x);
    case 4: return __fadd_rn(__fmul_rn(gy, v.w), v.y);
    default: return __fsub_rn(__fmul_rn(gy, v.w), v.y);
  }
}

// clip coordinates of vertex i: [v,1] . M (row-vector layout of full_proj_transform), summed left to right
__device__ __forceinline__ PV clip_vertex(const MeshParams& p, const float* cam, int i) {
  PV o;
  if (p.pos_kind == GAB200_MESH_POS_CLIP) {
    const float* v = p.verts + 4 * (int64_t)i;
    o.x = v[0]; o.y = v[1]; o.z = v[2]; o.w = v[3];
  } else {
    const float* v = p.verts + 3 * (int64_t)i;
    const float* M = cam + 16;
    float c[4];
#pragma unroll
    for (int j = 0; j < 4; j++)
      c[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], M[j]), __fmul_rn(v[1], M[4 + j])), __fmul_rn(v[2], M[8 + j])),
                       M[12 + j]);
    o.x = c[0]; o.y = c[1]; o.z = c[2]; o.w = c[3];
  }
  o.b0 = 0.f; o.b1 = 0.f;
  return o;
}

__device__ __forceinline__ bool inside_all(const PV& v, float gx, float gy) {
  bool in = v.w > 0.f;
#pragma unroll
  for (int k = 0; k < 6; k++) in = in && plane_dist(v, k, gx, gy) >= 0.f;
  return in;
}

__device__ __forceinline__ void snap(const PV& v, int W, int H, int& sx, int& sy) {
  const float X = __fmul_rn(__fadd_rn(__fdiv_rn(v.x, v.w), 1.f), 0.5f * (float)W);
  const float Y = __fmul_rn(__fadd_rn(__fdiv_rn(v.y, v.w), 1.f), 0.5f * (float)H);
  sx = __float2int_rn(__fmul_rn(X, 256.f));
  sy = __float2int_rn(__fmul_rn(Y, 256.f));
}

// signed doubled area of (a, b, p) in 1/256 px units: > 0 left of a->b in a y-down frame
__device__ __forceinline__ int64_t edge_fn(int ax, int ay, int bx, int by, int64_t px, int64_t py) {
  return (int64_t)(bx - ax) * (py - ay) - (int64_t)(by - ay) * (px - ax);
}

// A sample exactly on an edge belongs to the side the perturbation (+eps, +eps^2) moves it into: the two faces of a
// shared edge see it with opposite direction, so exactly one of them takes it (and one face only at a shared vertex).
__device__ __forceinline__ bool on_edge_owned(int dx, int dy) { return dy < 0 || (dy == 0 && dx > 0); }

__device__ __forceinline__ uint32_t depth_key(float z) {
  const uint32_t u = __float_as_uint(z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_depth(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ bool face_ok(const MeshParams& p, int f, int& i0, int& i1, int& i2) {
  i0 = p.faces[3 * (int64_t)f]; i1 = p.faces[3 * (int64_t)f + 1]; i2 = p.faces[3 * (int64_t)f + 2];
  return i0 >= 0 && i0 < p.V && i1 >= 0 && i1 < p.V && i2 >= 0 && i2 < p.V;
}

// Sub-triangle (A, B, C) of a polygon, oriented so that its area is positive; false if degenerate.
struct SubTri {
  int ax, ay, bx, by, cx, cy, ia, ib, ic;
  int64_t area;
  __device__ __forceinline__ bool init(const FacePoly& P, int j) {
    ia = 0; ib = j; ic = j + 1;
    ax = P.sx[0]; ay = P.sy[0]; bx = P.sx[j]; by = P.sy[j]; cx = P.sx[j + 1]; cy = P.sy[j + 1];
    area = edge_fn(ax, ay, bx, by, cx, cy);
    if (area == 0) return false;
    if (area < 0) {
      int t = bx; bx = cx; cx = t; t = by; by = cy; cy = t; t = ib; ib = ic; ic = t;
      area = -area;
    }
    return true;
  }
  // edge functions opposite A, B, C at (px, py); true if the sample is covered
  __device__ __forceinline__ bool cover(int64_t px, int64_t py, int64_t& e0, int64_t& e1, int64_t& e2) const {
    e0 = edge_fn(bx, by, cx, cy, px, py);
    e1 = edge_fn(cx, cy, ax, ay, px, py);
    e2 = edge_fn(ax, ay, bx, by, px, py);
    return (e0 > 0 || (e0 == 0 && on_edge_owned(cx - bx, cy - by))) &&
           (e1 > 0 || (e1 == 0 && on_edge_owned(ax - cx, ay - cy))) &&
           (e2 > 0 || (e2 == 0 && on_edge_owned(bx - ax, by - ay)));
  }
  __device__ __forceinline__ float depth(const FacePoly& P, int64_t e0, int64_t e1, int64_t e2) const {
    const float s = __fadd_rn(__fadd_rn(__fmul_rn(__ll2float_rn(e0), P.zw[ia]), __fmul_rn(__ll2float_rn(e1), P.zw[ib])),
                              __fmul_rn(__ll2float_rn(e2), P.zw[ic]));
    return __fdiv_rn(s, __ll2float_rn(area));
  }
};

__global__ void __launch_bounds__(128) mesh_setup_kernel(MeshParams p, const float* face_colors, float3 bg,
                                                         int lighting, FacePoly* polys, FaceEdges* edges,
                                                         float4* colors, uint64_t* tiles, int32_t* error_flag) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;   // record of (view, face): K F <= INT32_MAX
  if (t >= p.K * p.F) return;
  const int view = t / p.F, f = t - view * p.F;
  const float* cam = p.cam + (int64_t)view * GAB200_CAMERA_FLOATS;
  FacePoly P;
  P.n = 0;
  FaceEdges E;
  E.inside = 0; E.orient = 0;
#pragma unroll
  for (int k = 0; k < 3; k++) E.vx[k] = E.vy[k] = 0;
  float4 col = make_float4(1.f, 1.f, 1.f, 1.f);
  int idx[3];
  if (!face_ok(p, f, idx[0], idx[1], idx[2])) {
    if (error_flag) atomicOr(error_flag, 1);
  } else {
    PV a[MAXP], b[MAXP];
    for (int k = 0; k < 3; k++) {
      a[k] = clip_vertex(p, cam, idx[k]);
      a[k].b0 = k == 0 ? 1.f : 0.f;
      a[k].b1 = k == 1 ? 1.f : 0.f;
      if (inside_all(a[k], p.gx, p.gy)) {
        E.inside |= 1 << k;
        snap(a[k], p.W, p.H, E.vx[k], E.vy[k]);
      }
    }
    if (E.inside == 7) {
      const int64_t s = edge_fn(E.vx[0], E.vy[0], E.vx[1], E.vy[1], E.vx[2], E.vy[2]);
      E.orient = s > 0 ? 1 : (s < 0 ? -1 : 0);
    }
    // Sutherland-Hodgman against the six planes in a fixed order (skipped when every vertex is inside)
    int n = 3;
    if (E.inside != 7) {
      PV* src = a;
      PV* dst = b;
      for (int k = 0; k < 6 && n > 0; k++) {
        int m = 0;
        for (int i = 0; i < n; i++) {
          const PV& c = src[i];
          const PV& d = src[i + 1 < n ? i + 1 : 0];
          const float dc = plane_dist(c, k, p.gx, p.gy), dd = plane_dist(d, k, p.gx, p.gy);
          if (dc >= 0.f) dst[m++] = c;
          if ((dc >= 0.f) != (dd >= 0.f) && m < MAXP) {
            const float t = __fdiv_rn(dc, __fsub_rn(dc, dd));
            PV o;
            o.x = __fadd_rn(c.x, __fmul_rn(t, __fsub_rn(d.x, c.x)));
            o.y = __fadd_rn(c.y, __fmul_rn(t, __fsub_rn(d.y, c.y)));
            o.z = __fadd_rn(c.z, __fmul_rn(t, __fsub_rn(d.z, c.z)));
            o.w = __fadd_rn(c.w, __fmul_rn(t, __fsub_rn(d.w, c.w)));
            o.b0 = __fadd_rn(c.b0, __fmul_rn(t, __fsub_rn(d.b0, c.b0)));
            o.b1 = __fadd_rn(c.b1, __fmul_rn(t, __fsub_rn(d.b1, c.b1)));
            dst[m++] = o;
          }
        }
        n = m;
        PV* t = src; src = dst; dst = t;
      }
      if (src != a)
        for (int i = 0; i < n; i++) a[i] = src[i];
    }
    bool ok = n >= 3;
    for (int i = 0; i < n; i++) ok = ok && a[i].w > 0.f;
    if (ok) {
      P.n = n;
      int xmin = INT_MAX, xmax = INT_MIN, ymin = INT_MAX, ymax = INT_MIN;
      for (int i = 0; i < n; i++) {
        snap(a[i], p.W, p.H, P.sx[i], P.sy[i]);
        P.zw[i] = __fdiv_rn(a[i].z, a[i].w);
        P.b0[i] = a[i].b0; P.b1[i] = a[i].b1;
        P.iw[i] = __fdiv_rn(1.f, a[i].w);
        xmin = min(xmin, P.sx[i]); xmax = max(xmax, P.sx[i]);
        ymin = min(ymin, P.sy[i]); ymax = max(ymax, P.sy[i]);
      }
      // centre 256 c + 128 inside [xmin, xmax]: arithmetic shifts floor
      P.c0 = max(-((128 - xmin) >> 8), 0); P.c1 = min((xmax - 128) >> 8, p.W - 1);
      P.r0 = max(-((128 - ymin) >> 8), 0); P.r1 = min((ymax - 128) >> 8, p.H - 1);
    }
    if (p.pos_kind == GAB200_MESH_POS_WORLD) {
      // face normal in the OpenGL camera frame (rows 1, 2 of the view transform negated), 'front' light on +z
      const float* Wv = cam;
      float c[3][3];
      for (int k = 0; k < 3; k++) {
        const float* v = p.verts + 3 * (int64_t)idx[k];
        for (int j = 0; j < 3; j++) {
          const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], Wv[j]), __fmul_rn(v[1], Wv[4 + j])),
                                              __fmul_rn(v[2], Wv[8 + j])), Wv[12 + j]);
          c[k][j] = j == 0 ? s : -s;
        }
      }
      float diffuse = 1.f;
      if (lighting == GAB200_MESH_LIGHT_FRONT) {
        const float e1x = c[1][0] - c[0][0], e1y = c[1][1] - c[0][1], e1z = c[1][2] - c[0][2];
        const float e2x = c[2][0] - c[0][0], e2y = c[2][1] - c[0][1], e2z = c[2][2] - c[0][2];
        const float nx = e1y * e2z - e1z * e2y, ny = e1z * e2x - e1x * e2z, nz = e1x * e2y - e1y * e2x;
        const float len = sqrtf(fmaxf(nx * nx + ny * ny + nz * nz, 1e-20f));
        diffuse = fminf(fmaxf(nz / len, 0.f), 1.f);
      }
      if (face_colors) {
        col.x = face_colors[3 * (int64_t)f] * diffuse;
        col.y = face_colors[3 * (int64_t)f + 1] * diffuse;
        col.z = face_colors[3 * (int64_t)f + 2] * diffuse;
      } else {
        col.x = col.y = col.z = diffuse;
      }
    }
  }
  uint64_t nt = 0;
  if (P.n > 0 && P.c1 >= P.c0 && P.r1 >= P.r0)
    nt = (uint64_t)((P.c1 - P.c0) / 8 + 1) * (uint64_t)((P.r1 - P.r0) / 4 + 1);
  polys[t] = P;
  edges[t] = E;
  colors[t] = col;
  tiles[t] = nt;
}

// Persistent warps over the (view, face, 8x4 tile) work items: warp k takes the k-th equal share of the items in order,
// finds the record of its first item by one binary search (the first t with offsets[t] > w) and walks the records
// forward.  Record t is face t mod F of view t / F; its key carries the face index and lands in that view's map.
__global__ void __launch_bounds__(256) mesh_raster_kernel(int F, int KF, int W, int64_t HW,
                                                          const FacePoly* __restrict__ polys,
                                                          const uint64_t* __restrict__ offsets,
                                                          unsigned long long* __restrict__ winner) {
  const int lane = threadIdx.x & 31;
  const uint64_t total = offsets[KF - 1];
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  const uint64_t per = (total + nwarps - 1) / nwarps;
  uint64_t w = ((uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * per;
  const uint64_t wend = min(total, w + per);
  if (w >= wend) return;
  int lo = 0, hi = KF - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] > w) hi = mid; else lo = mid + 1;
  }
  int t = lo;
  int view = t / F, f = t - view * F;
  unsigned long long* map = winner + view * HW;
  uint64_t base = t > 0 ? offsets[t - 1] : 0ull, end = offsets[t];
  for (; w < wend; w++) {
    if (w >= end) {
      do {
        base = end;
        end = offsets[++t];
      } while (w >= end);
      view = t / F;
      f = t - view * F;
      map = winner + view * HW;
    }
    const uint64_t local = w - base;
    const FacePoly& P = polys[t];
    const int c0 = P.c0, r0 = P.r0;
    const uint64_t ntx = (uint64_t)((P.c1 - c0) / 8 + 1);
    const int c = c0 + (int)(local % ntx) * 8 + (lane & 7);
    const int r = r0 + (int)(local / ntx) * 4 + (lane >> 3);
    if (c > P.c1 || r > P.r1) continue;
    const int64_t px = 256 * (int64_t)c + 128, py = 256 * (int64_t)r + 128;
    uint64_t best = EMPTY;
    for (int j = 1; j + 1 < P.n; j++) {
      SubTri T;
      if (!T.init(P, j)) continue;
      int64_t e0, e1, e2;
      if (!T.cover(px, py, e0, e1, e2)) continue;
      const uint64_t key = ((uint64_t)depth_key(T.depth(P, e0, e1, e2)) << 32) | (uint32_t)f;
      best = key < best ? key : best;
    }
    if (best != EMPTY) atomicMin(map + (int64_t)r * W + c, (unsigned long long)best);
  }
}

// The winner map from an nvdiffrast-layout rast tensor [H,W,4] (z/w in channel 2, id + 1 in channel 3).
__global__ void mesh_keys_from_rast_kernel(int n, int F, const float* __restrict__ rast, uint64_t* __restrict__ winner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float id1 = rast[4 * (int64_t)i + 3];
  uint64_t k = EMPTY;
  if (id1 >= 1.f && id1 <= (float)F) k = ((uint64_t)depth_key(rast[4 * (int64_t)i + 2]) << 32) | (uint32_t)((int)id1 - 1);
  winner[i] = k;
}

// One thread per (view, face): which of its edges are screen-space silhouettes -- a mesh boundary, or the face across it lies
// on the face's side of the edge's projected line (the opposite vertex of the neighbour read from its own record:
// the same snapped position a projection here would give).  Edges with a vertex outside the clip volume, and every
// edge of a face with such a vertex (orient 0), never are.
__global__ void __launch_bounds__(128) mesh_silhouette_kernel(MeshParams p, FaceEdges* all_edges) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.K * p.F) return;
  const int view = t / p.F, T = t - view * p.F;
  FaceEdges* edges = all_edges + (int64_t)view * p.F;   // this view's records
  const FaceEdges E = edges[T];
  int a[3], n[3];
  if (E.orient == 0 || !face_ok(p, T, a[0], a[1], a[2])) return;
  int sil = 0;
  for (int k = 0; k < 3; k++) {
    const int k1 = k == 2 ? 0 : k + 1;
    if (((E.inside >> k) & 1) == 0 || ((E.inside >> k1) & 1) == 0) continue;
    const int N = p.adj[3 * (int64_t)T + k];
    if (N == -1) { sil |= 1 << k; continue; }
    if (N < 0 || N >= p.F || !face_ok(p, N, n[0], n[1], n[2])) continue;
    int j = -1;
    for (int i = 2; i >= 0; i--)
      if (n[i] != a[k] && n[i] != a[k1]) j = i;
    if (j < 0) continue;
    const FaceEdges EN = edges[N];
    if (((EN.inside >> j) & 1) == 0) continue;
    const int64_t s = edge_fn(E.vx[k], E.vy[k], E.vx[k1], E.vy[k1], EN.vx[j], EN.vy[j]);
    if ((s > 0 && E.orient > 0) || (s < 0 && E.orient < 0)) sil |= 1 << k;
  }
  edges[T].inside = E.inside | (sil << 3);
}

// The blend of the pair (q, n) that moves q: the weight q moves toward n by, or 0.  horizontal: n is q's left / right
// neighbour.  Both pixels of a pair evaluate the same function, so the two sides always agree.
__device__ float pair_weight(const FaceEdges* __restrict__ edges, int qc, int qr, uint64_t kq,
                             int nc, int nr, uint64_t kn, bool horizontal) {
  if (kq == kn) return 0.f;
  const bool q_occ = kq < kn;
  const uint64_t ko = q_occ ? kq : kn;
  const int T = (int)(uint32_t)ko;
  const int ac = q_occ ? qc : nc, ar = q_occ ? qr : nr, bc = q_occ ? nc : qc, br = q_occ ? nr : qr;
  const FaceEdges E = edges[T];
  const int64_t ax = 256 * (int64_t)ac + 128, ay = 256 * (int64_t)ar + 128;
  const int64_t bx = 256 * (int64_t)bc + 128, by = 256 * (int64_t)br + 128;
  float tbest = 2.f;
  for (int k = 0; k < 3; k++) {
    const int k1 = k == 2 ? 0 : k + 1;
    const int dx = E.vx[k1] - E.vx[k], dy = E.vy[k1] - E.vy[k];
    if ((abs(dx) <= abs(dy)) != horizontal) continue;
    if (((E.inside >> (3 + k)) & 1) == 0) continue;
    const int64_t ea = edge_fn(E.vx[k], E.vy[k], E.vx[k1], E.vy[k1], ax, ay);
    const int64_t eb = edge_fn(E.vx[k], E.vy[k], E.vx[k1], E.vy[k1], bx, by);
    if (ea == eb) continue;
    const float t = __fdiv_rn(__ll2float_rn(ea), __ll2float_rn(ea - eb));
    if (!(t >= 0.f && t <= 1.f)) continue;
    if (horizontal) {
      if (ay < min(E.vy[k], E.vy[k1]) || ay > max(E.vy[k], E.vy[k1])) continue;
    } else {
      if (ax < min(E.vx[k], E.vx[k1]) || ax > max(E.vx[k], E.vx[k1])) continue;
    }
    tbest = t < tbest ? t : tbest;
  }
  if (tbest > 1.f) return 0.f;
  if (tbest < 0.5f) return q_occ ? __fsub_rn(0.5f, tbest) : 0.f;
  if (tbest > 0.5f) return q_occ ? 0.f : __fsub_rn(tbest, 0.5f);
  return 0.f;
}

__device__ __forceinline__ uint32_t quantize_u8(float c) {  // render.py's mul(255).add_(0.5).clamp_(0, 255), truncated
  return __float2uint_rz(fminf(fmaxf(__fadd_rn(__fmul_rn(c, 255.f), 0.5f), 0.f), 255.f));
}

struct ResolveOut {
  int antialias, base_kind, channels;
  float3 bg;
  const void* base;
  const float* opacity;
  const float* in_color;
  uint8_t* out_u8;
  float* out_float;
  float* out_rgba;
  float* out_rast;
  float* out_color;
};

// One thread per (view, pixel), view = blockIdx.z.  Only base and out_u8 have a view dimension: the other outputs
// exist for single-view calls only.  VIEWER: out_u8 quantised as the local viewer's export (GAB200_QUANTIZE_VIEWER).
template <bool VIEWER>
__global__ void __launch_bounds__(256) mesh_resolve_kernel(MeshParams p, ResolveOut o,
                                                           const FacePoly* __restrict__ all_polys,
                                                           const FaceEdges* __restrict__ all_edges,
                                                           const float4* __restrict__ all_colors,
                                                           const uint64_t* __restrict__ all_winner) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (c >= p.W) return;
  const int64_t pix = (int64_t)r * p.W + c, HW = (int64_t)p.W * p.H;
  const int64_t view = blockIdx.z;
  const FacePoly* __restrict__ polys = all_polys + view * p.F;
  const FaceEdges* __restrict__ edges = all_edges + view * p.F;
  const float4* __restrict__ colors = all_colors + view * p.F;
  const uint64_t* __restrict__ winner = all_winner + view * HW;
  const uint64_t kq = winner[pix];
  // neighbours in the fixed order left, right, up, down
  float wgt[4] = {0.f, 0.f, 0.f, 0.f};
  int64_t npix[4] = {pix, pix, pix, pix};
  if (o.antialias) {
    const int nc[4] = {c - 1, c + 1, c, c}, nr[4] = {r, r, r - 1, r + 1};
#pragma unroll
    for (int j = 0; j < 4; j++) {
      if (nc[j] < 0 || nc[j] >= p.W || nr[j] < 0 || nr[j] >= p.H) continue;
      npix[j] = (int64_t)nr[j] * p.W + nc[j];
      wgt[j] = pair_weight(edges, c, r, kq, nc[j], nr[j], winner[npix[j]], j < 2);
    }
  }
  if (o.in_color) {  // antialias of a caller image [H,W,C]
    for (int ch = 0; ch < o.channels; ch++) {
      const float cq = o.in_color[pix * o.channels + ch];
      float acc = cq;
#pragma unroll
      for (int j = 0; j < 4; j++)
        if (wgt[j] != 0.f) acc = __fadd_rn(acc, __fmul_rn(wgt[j], __fsub_rn(o.in_color[npix[j] * o.channels + ch], cq)));
      o.out_color[pix * o.channels + ch] = acc;
    }
  }
  if (o.out_rast) {
    float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (kq != EMPTY) {
      const int f = (int)(uint32_t)kq;
      const FacePoly& P = polys[f];
      const int64_t px = 256 * (int64_t)c + 128, py = 256 * (int64_t)r + 128;
      for (int j = 1; j + 1 < P.n; j++) {
        SubTri T;
        if (!T.init(P, j)) continue;
        int64_t e0, e1, e2;
        if (!T.cover(px, py, e0, e1, e2)) continue;
        const float ar = __ll2float_rn(T.area);
        const float qa = __fmul_rn(__fdiv_rn(__ll2float_rn(e0), ar), P.iw[T.ia]);
        const float qb = __fmul_rn(__fdiv_rn(__ll2float_rn(e1), ar), P.iw[T.ib]);
        const float qc = __fmul_rn(__fdiv_rn(__ll2float_rn(e2), ar), P.iw[T.ic]);
        const float s = qa + qb + qc;
        rv.x = (qa * P.b0[T.ia] + qb * P.b0[T.ib] + qc * P.b0[T.ic]) / s;
        rv.y = (qa * P.b1[T.ia] + qb * P.b1[T.ib] + qc * P.b1[T.ic]) / s;
        break;
      }
      rv.z = key_depth((uint32_t)(kq >> 32));
      rv.w = (float)(f + 1);
    }
    reinterpret_cast<float4*>(o.out_rast)[pix] = rv;
  }
  if (!o.out_rgba && !o.out_u8 && !o.out_float) return;
  auto rgba_of = [&](uint64_t k) {
    return k == EMPTY ? make_float4(o.bg.x, o.bg.y, o.bg.z, 0.f) : colors[(uint32_t)k];
  };
  const float4 cq = rgba_of(kq);
  float4 acc = cq;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    if (wgt[j] == 0.f) continue;
    const float4 cn = rgba_of(winner[npix[j]]);
    acc.x = __fadd_rn(acc.x, __fmul_rn(wgt[j], __fsub_rn(cn.x, cq.x)));
    acc.y = __fadd_rn(acc.y, __fmul_rn(wgt[j], __fsub_rn(cn.y, cq.y)));
    acc.z = __fadd_rn(acc.z, __fmul_rn(wgt[j], __fsub_rn(cn.z, cq.z)));
    acc.w = __fadd_rn(acc.w, __fmul_rn(wgt[j], __fsub_rn(cn.w, cq.w)));
  }
  if (o.out_rgba) reinterpret_cast<float4*>(o.out_rgba)[pix] = acc;
  if (!o.out_u8 && !o.out_float) return;
  // rgb * a * o + base * (a * (1 - o) + (1 - a)), torch's evaluation order, every op rounded
  const float op = o.opacity[0], omo = o.opacity[1];
  const float a = acc.w;
  const float keep = __fadd_rn(__fmul_rn(a, omo), __fsub_rn(1.f, a));
  const float rgb[3] = {acc.x, acc.y, acc.z};
  uint32_t q[3];
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    float b;
    if (o.base_kind == GAB200_MESH_BASE_U8_CHW)
      b = __fdiv_rn((float)static_cast<const uint8_t*>(o.base)[(3 * view + ch) * HW + pix], 255.f);
    else
      b = static_cast<const float*>(o.base)[(3 * view + ch) * HW + pix];
    const float v = __fadd_rn(__fmul_rn(__fmul_rn(rgb[ch], a), op), __fmul_rn(b, keep));
    if (o.out_float) o.out_float[ch * HW + pix] = v;
    q[ch] = VIEWER ? quantize_u8_viewer(v) : quantize_u8(v);
  }
  if (o.out_u8) {
    uint8_t* out = o.out_u8 + 3 * (view * HW + pix);
    out[0] = (uint8_t)q[0];
    out[1] = (uint8_t)q[1];
    out[2] = (uint8_t)q[2];
  }
}

struct MeshScratch {
  FacePoly* polys;
  FaceEdges* edges;
  float4* colors;
  uint64_t* tiles;
  uint64_t* offsets;
  uint64_t* winner;
  void* scan_temp;
  size_t scan_bytes;
};

size_t scan_temp_bytes_u64(int F) {
  size_t bytes = 0;
  cub::DeviceScan::InclusiveSum(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, F);
  return bytes;
}

// K views: K F face records (K = 1: the single-view layout) and K winner maps
MeshScratch carve_mesh(void* base, int K, int F, int W, int H) {
  const int KF = K * F;
  Carver cv(base);
  MeshScratch s;
  s.polys = cv.take<FacePoly>(KF);
  s.edges = cv.take<FaceEdges>(KF);
  s.colors = cv.take<float4>(KF);
  s.tiles = cv.take<uint64_t>(KF);
  s.offsets = cv.take<uint64_t>(KF);
  s.winner = cv.take<uint64_t>((size_t)K * W * H);
  s.scan_bytes = scan_temp_bytes_u64(KF);
  s.scan_temp = cv.take<char>(s.scan_bytes);
  return s;
}

}  // namespace

size_t mesh_scratch_bytes(int K, int F, int W, int H) {
  Carver cv(nullptr);
  const int KF = K * F;
  cv.take<FacePoly>(KF);
  cv.take<FaceEdges>(KF);
  cv.take<float4>(KF);
  cv.take<uint64_t>(KF);
  cv.take<uint64_t>(KF);
  cv.take<uint64_t>((size_t)K * W * H);
  cv.take<char>(scan_temp_bytes_u64(KF));
  return cv.bytes();
}

cudaError_t launch_mesh_render(const gab200_mesh_args& a, int K, cudaStream_t stream) {
  MeshScratch s = carve_mesh(a.scratch, K, a.F, a.width, a.height);
  MeshParams p;
  p.V = a.V; p.F = a.F; p.W = a.width; p.H = a.height; p.pos_kind = a.pos_kind; p.K = K;
  p.verts = a.verts; p.faces = a.faces; p.adj = a.adjacency; p.cam = a.camera;
  p.gx = 65536.f / (float)a.width;  // IEEE division on the host, as the oracle's float32 division
  p.gy = 65536.f / (float)a.height;
  const float3 bg = make_float3(a.background[0], a.background[1], a.background[2]);
  const int KF = K * a.F;
  mesh_setup_kernel<<<(KF + 127) / 128, 128, 0, stream>>>(p, a.face_colors, bg, a.lighting, s.polys, s.edges,
                                                          s.colors, s.tiles, a.error_flag);
  count_launch();
  if (a.antialias) {
    mesh_silhouette_kernel<<<(KF + 127) / 128, 128, 0, stream>>>(p, s.edges);
    count_launch();
  }
  const int64_t HW = (int64_t)a.width * a.height;
  if (a.in_rast) {   // single-view calls only
    mesh_keys_from_rast_kernel<<<(unsigned)((HW + 255) / 256), 256, 0, stream>>>((int)HW, a.F, a.in_rast, s.winner);
    count_launch();
  } else {
    cudaError_t e = cudaMemsetAsync(s.winner, 0xff, K * HW * sizeof(uint64_t), stream);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::InclusiveSum(s.scan_temp, s.scan_bytes, s.tiles, s.offsets, KF, stream);
    if (e != cudaSuccess) return e;
    count_launch();
    mesh_raster_kernel<<<GAB_NUM_SMS * 8, 256, 0, stream>>>(a.F, KF, a.width, HW, s.polys, s.offsets,
                                                            reinterpret_cast<unsigned long long*>(s.winner));
    count_launch();
  }
  ResolveOut o;
  o.antialias = a.antialias; o.base_kind = a.base_kind; o.channels = a.channels;
  o.bg = bg; o.base = a.base; o.opacity = a.opacity; o.in_color = a.in_color;
  o.out_u8 = a.out_u8; o.out_float = a.out_float; o.out_rgba = a.out_rgba; o.out_rast = a.out_rast;
  o.out_color = a.out_color;
  const dim3 grid((a.width + 255) / 256, a.height, K);
  if (a.quantize == GAB200_QUANTIZE_VIEWER)
    mesh_resolve_kernel<true><<<grid, 256, 0, stream>>>(p, o, s.polys, s.edges, s.colors, s.winner);
  else
    mesh_resolve_kernel<false><<<grid, 256, 0, stream>>>(p, o, s.polys, s.edges, s.colors, s.winner);
  count_launch();
  return cudaPeekAtLastError();
}

}  // namespace gab
