// flame.cu -- FLAME head posing (blendshapes + linear blend skinning) for one timestep, forward and backward.
// Replaces FlameHead.forward + lbs (flame_model/flame.py:485-558, flame_model/lbs.py:25-304) as
// select_mesh_by_timestep calls it (scene/flame_gaussian_model.py:117-135).  See include/gab200_rasterizer.h for the
// semantics; the layout of the prepared scratch is private to this file.
//
// Per frame, two launches each way:
//   flame_joints_kernel           1 CTA   J = J_base + JS.expr; Rodrigues x5; rigid chain -> A (5 x 3x4); pose feature
//   flame_skin_kernel             3V/96   v_shaped = v_base + E.expr; v_posed = v_shaped + P^T.pf; verts = (sum w A).v
//   flame_skin_backward_kernel    3V/96   same basis reads (kept in registers) + per-CTA partial sums of dA, dpf,
//                                         E^T.dv_shaped, dtranslation; zeroes the gradient rows != t
//   flame_joints_backward_kernel  1 CTA   sums the partials in CTA order, chain + Rodrigues backward, JS^T.dJ
// A CTA covers 32 vertices (96 coordinates) with 8 warp-triples splitting the n_expr + 36 basis components, so the
// ~8.5 MB basis read of a full FLAME head (V = 5143) runs on 161 CTAs with ~18 loads in flight per thread.
// The joint-chain arithmetic (a few hundred flops) runs in double and is rounded to float once.
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

#define FL_J GAB200_FLAME_J
#define FL_PB GAB200_FLAME_POSE_BASIS
#define FL_TV 32                      // vertices per CTA
#define FL_COLS (3 * FL_TV)           // coordinates per CTA
#define FL_S 8                        // component slices per CTA (one warp-triple each)
#define FL_THREADS (FL_COLS * FL_S)   // 768
#define FL_ME ((GAB200_FLAME_MAX_EXPR + FL_S - 1) / FL_S)   // expression components per thread (13)
#define FL_MP ((FL_PB + FL_S - 1) / FL_S)                   // pose-basis components per thread (5)
// per-CTA partial record of the backward: dA [60] | dpose_feature [36] | dtranslation [3] | E^T.dv_shaped [n_expr]
#define FL_P_A 0
#define FL_P_PF 60
#define FL_P_TR 96
#define FL_P_EX 99
// frame record (GAB200_FLAME_FRAME_FLOATS): A [60] | pose feature [36] | posed joints [15]
#define FL_F_A 0
#define FL_F_PF 60
#define FL_F_J 96

struct FlameView {
  float* v_base;    // [3V]
  float* basis;     // [n_expr, 3V] expression basis, component-major
  float* J_base;    // [15]
  float* JS;        // [15, n_expr]
  float* partials;  // [n_blocks, pstride]
  int n_blocks, pstride;
  size_t bytes;
};

static FlameView carve_flame(void* p, int V, int NE) {
  Carver cv(p);
  FlameView f;
  f.n_blocks = (V + FL_TV - 1) / FL_TV;
  f.pstride = (FL_P_EX + NE + 3) & ~3;
  f.v_base = cv.take<float>(3 * (size_t)V);
  f.basis = cv.take<float>((size_t)NE * 3 * V);
  f.J_base = cv.take<float>(15);
  f.JS = cv.take<float>(15 * (size_t)NE);
  f.partials = cv.take<float>((size_t)f.n_blocks * f.pstride);
  f.bytes = cv.bytes();
  return f;
}

size_t flame_scratch_bytes(int V, int NE) { return carve_flame(nullptr, V, NE).bytes; }

struct FlameParents {
  int p[FL_J];
};

// ---- prepare ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) flame_prepare_vertex_kernel(int V, int NS, int NE, const float* __restrict__ v_template,
                                                                   const float* __restrict__ shapedirs,
                                                                   const float* __restrict__ shape,
                                                                   const float* __restrict__ static_offset,
                                                                   float* __restrict__ v_base, float* __restrict__ basis) {
  const int n3 = 3 * V;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n3) return;
  const float* row = shapedirs + (size_t)c * (NS + NE);
  double acc = 0.0;
  for (int l = 0; l < NS; l++) acc += (double)row[l] * (double)shape[l];
  acc += (double)v_template[c];
  if (static_offset != nullptr) acc += (double)static_offset[c];
  v_base[c] = (float)acc;
  for (int e = 0; e < NE; e++) basis[(size_t)e * n3 + c] = row[NS + e];
}

// J_base (blockIdx.y == 0) and JS (blockIdx.y = 1 + e): one regressor row (joint j, axis k = blockIdx.x) per CTA
__global__ void __launch_bounds__(256) flame_prepare_joint_kernel(int V, int NE, const float* __restrict__ J_regressor,
                                                                  const float* __restrict__ v_base,
                                                                  const float* __restrict__ basis,
                                                                  float* __restrict__ J_base, float* __restrict__ JS) {
  __shared__ double red[256];
  const int jk = blockIdx.x, j = jk / 3, k = jk % 3, col = blockIdx.y;
  const int n3 = 3 * V;
  const float* src = col == 0 ? v_base : basis + (size_t)(col - 1) * n3;
  double acc = 0.0;
  for (int v = threadIdx.x; v < V; v += blockDim.x) acc += (double)J_regressor[(size_t)j * V + v] * (double)src[3 * v + k];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (col == 0)
      J_base[jk] = (float)red[0];
    else
      JS[(size_t)jk * NE + col - 1] = (float)red[0];
  }
}

// ---- joint chain (double) -----------------------------------------------------------------------------------------
struct Rod {   // Rodrigues of lbs.py:25-57 with what its backward needs
  double a[3], th, d[3], s, c, K[9], K2[9], R[9];
};

__device__ void rodrigues(const double r[3], Rod& o) {
  for (int i = 0; i < 3; i++) o.a[i] = r[i] + 1e-8;   // torch.norm(rot_vecs + 1e-8)
  o.th = sqrt(o.a[0] * o.a[0] + o.a[1] * o.a[1] + o.a[2] * o.a[2]);
  for (int i = 0; i < 3; i++) o.d[i] = r[i] / o.th;
  o.s = sin(o.th);
  o.c = cos(o.th);
  const double x = o.d[0], y = o.d[1], z = o.d[2];
  const double K[9] = {0, -z, y, z, 0, -x, -y, x, 0};
  for (int i = 0; i < 9; i++) o.K[i] = K[i];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double m = 0;
      for (int l = 0; l < 3; l++) m += K[3 * i + l] * K[3 * l + j];
      o.K2[3 * i + j] = m;
    }
  for (int i = 0; i < 9; i++) o.R[i] = (i % 4 == 0 ? 1.0 : 0.0) + o.s * o.K[i] + (1.0 - o.c) * o.K2[i];
}

__device__ void rodrigues_backward(const double r[3], const Rod& o, const double dR[9], double dr[3]) {
  double gs = 0, gomc = 0;
  for (int i = 0; i < 9; i++) {
    gs += dR[i] * o.K[i];
    gomc += dR[i] * o.K2[i];
  }
  // d<dR, K^2>/dK = dR K^T + K^T dR
  double dK[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double m = 0;
      for (int l = 0; l < 3; l++) m += dR[3 * i + l] * o.K[3 * j + l] + o.K[3 * l + i] * dR[3 * l + j];
      dK[3 * i + j] = o.s * dR[3 * i + j] + (1.0 - o.c) * m;
    }
  double dth = gs * o.c + gomc * o.s;   // s = sin(th), (1 - c) = 1 - cos(th)
  const double dd[3] = {dK[7] - dK[5], dK[2] - dK[6], dK[3] - dK[1]};
  const double th2 = o.th * o.th;
  for (int i = 0; i < 3; i++) {
    dr[i] = dd[i] / o.th;
    dth -= dd[i] * r[i] / th2;
  }
  for (int i = 0; i < 3; i++) dr[i] += dth * o.a[i] / o.th;
}

struct Chain {
  double J[FL_J][3];      // rest joints
  double pose[3 * FL_J];  // full_pose
  Rod rod[FL_J];
  double rel[FL_J][3];
  double Rc[FL_J][9], tc[FL_J][3];   // global transforms
};

struct ChainGrad {
  double dRc[FL_J][9], dtc[FL_J][3], dR[FL_J][9], drel[FL_J][3], gJ[FL_J][3];
};

__device__ void load_pose(int t, const float* rot, const float* neck, const float* jaw, const float* eyes,
                          double pose[3 * FL_J]) {
  for (int k = 0; k < 3; k++) {
    pose[k] = rot[3 * t + k];
    pose[3 + k] = neck[3 * t + k];
    pose[6 + k] = jaw[3 * t + k];
  }
  for (int k = 0; k < 6; k++) pose[9 + k] = eyes[6 * t + k];
}

__device__ void chain_forward(Chain& ch, const FlameParents& par) {   // lbs.py:254-304
  for (int i = 0; i < FL_J; i++) {
    rodrigues(ch.pose + 3 * i, ch.rod[i]);
    for (int k = 0; k < 3; k++) ch.rel[i][k] = ch.J[i][k] - (i == 0 ? 0.0 : ch.J[par.p[i]][k]);
  }
  for (int i = 0; i < 9; i++) ch.Rc[0][i] = ch.rod[0].R[i];
  for (int k = 0; k < 3; k++) ch.tc[0][k] = ch.rel[0][k];
  for (int i = 1; i < FL_J; i++) {
    const int p = par.p[i];
    const double* Rp = ch.Rc[p];
    const double* Ri = ch.rod[i].R;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++)
        ch.Rc[i][3 * r + c] = Rp[3 * r] * Ri[c] + Rp[3 * r + 1] * Ri[3 + c] + Rp[3 * r + 2] * Ri[6 + c];
      ch.tc[i][r] = Rp[3 * r] * ch.rel[i][0] + Rp[3 * r + 1] * ch.rel[i][1] + Rp[3 * r + 2] * ch.rel[i][2] + ch.tc[p][r];
    }
  }
}

__global__ void __launch_bounds__(32) flame_joints_kernel(int T, int NE, FlameParents par, const int32_t* __restrict__ tptr,
                                                          const float* __restrict__ expr, const float* __restrict__ rot,
                                                          const float* __restrict__ neck, const float* __restrict__ jaw,
                                                          const float* __restrict__ eyes, const float* __restrict__ trans,
                                                          const float* __restrict__ J_base, const float* __restrict__ JS,
                                                          float* __restrict__ frame) {
  const int t = *tptr;
  if (t < 0 || t >= T) return;
  __shared__ double sJ[15];
  if (threadIdx.x < 15) {
    const float* js = JS + (size_t)threadIdx.x * NE;
    const float* ex = expr + (size_t)t * NE;
    double acc = J_base[threadIdx.x];
    for (int e = 0; e < NE; e++) acc += (double)js[e] * (double)ex[e];
    sJ[threadIdx.x] = acc;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  __shared__ Chain ch;   // single-thread work: shared memory keeps the double arrays out of registers and local memory
  for (int i = 0; i < 15; i++) ch.J[i / 3][i % 3] = sJ[i];
  load_pose(t, rot, neck, jaw, eyes, ch.pose);
  chain_forward(ch, par);
  for (int i = 0; i < FL_J; i++) {
    for (int r = 0; r < 3; r++) {
      double rj = 0;
      for (int c = 0; c < 3; c++) {
        frame[FL_F_A + 12 * i + 4 * r + c] = (float)ch.Rc[i][3 * r + c];
        rj += ch.Rc[i][3 * r + c] * ch.J[i][c];
      }
      frame[FL_F_A + 12 * i + 4 * r + 3] = (float)(ch.tc[i][r] - rj);   // rel_transforms: t - R J
      frame[FL_F_J + 3 * i + r] = (float)(ch.tc[i][r] + (double)trans[3 * t + r]);
    }
    if (i > 0)
      for (int m = 0; m < 9; m++) frame[FL_F_PF + 9 * (i - 1) + m] = (float)(ch.rod[i].R[m] - (m % 4 == 0 ? 1.0 : 0.0));
  }
}

// ---- skinning -----------------------------------------------------------------------------------------------------
// This thread's share of the basis for coordinate c: expression components y, y+8, ... and pose components likewise.
__device__ __forceinline__ void load_basis(int c, int n3, int y, int NE, const float* __restrict__ basis,
                                           const float* __restrict__ posedirs, float ev[FL_ME], float pv[FL_MP]) {
  const bool in = c < n3;
#pragma unroll
  for (int i = 0; i < FL_ME; i++) {
    const int e = y + i * FL_S;
    ev[i] = (in && e < NE) ? __ldg(basis + (size_t)e * n3 + c) : 0.f;
  }
#pragma unroll
  for (int i = 0; i < FL_MP; i++) {
    const int p = y + i * FL_S;
    pv[i] = (in && p < FL_PB) ? __ldg(posedirs + (size_t)p * n3 + c) : 0.f;
  }
}

struct SkinShared {
  float expr[GAB200_FLAME_MAX_EXPR];
  float pf[FL_PB];
  float A[60];
  float acc[2][FL_S][FL_COLS];
  float vp[FL_COLS];
};

// stages expr[t], the pose feature and A; returns v_shaped / v_posed of coordinate x of this CTA's tile in sh.vp
// (and v_shaped through *vs_out for the row-0 threads)
__device__ __forceinline__ void skin_front(SkinShared& sh, int t, int NE, int n3, const float* __restrict__ expr,
                                           const float* __restrict__ frame, const float* __restrict__ v_base,
                                           const float ev[FL_ME], const float pv[FL_MP], float* vs_out) {
  const int x = threadIdx.x, y = threadIdx.y, tid = y * FL_COLS + x;
  if (tid < NE) sh.expr[tid] = expr[(size_t)t * NE + tid];
  if (tid < FL_PB) sh.pf[tid] = frame[FL_F_PF + tid];
  if (tid < 60) sh.A[tid] = frame[FL_F_A + tid];
  __syncthreads();
  float ae = 0.f, ap = 0.f;
#pragma unroll
  for (int i = 0; i < FL_ME; i++) {
    const int e = y + i * FL_S;
    if (e < NE) ae = fmaf(ev[i], sh.expr[e], ae);
  }
#pragma unroll
  for (int i = 0; i < FL_MP; i++) {
    const int p = y + i * FL_S;
    if (p < FL_PB) ap = fmaf(pv[i], sh.pf[p], ap);
  }
  sh.acc[0][y][x] = ae;
  sh.acc[1][y][x] = ap;
  __syncthreads();
  const int c = blockIdx.x * FL_COLS + x;
  if (y == 0) {
    float se = 0.f, sp = 0.f;
#pragma unroll
    for (int s = 0; s < FL_S; s++) {
      se += sh.acc[0][s][x];
      sp += sh.acc[1][s][x];
    }
    const float vs = c < n3 ? v_base[c] + se : 0.f;
    *vs_out = vs;
    sh.vp[x] = vs + sp;
  }
  __syncthreads();
}

// T_v = sum_j w_j A_j (3x4), lbs.py:182-185
__device__ __forceinline__ void blend_transform(const float* __restrict__ w, const float* A, float Tv[12]) {
#pragma unroll
  for (int m = 0; m < 12; m++) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < FL_J; j++) s = fmaf(w[j], A[12 * j + m], s);
    Tv[m] = s;
  }
}

__global__ void __launch_bounds__(FL_THREADS, 2) flame_skin_kernel(int V, int T, int NE, const int32_t* __restrict__ tptr,
                                                                const float* __restrict__ expr,
                                                                const float* __restrict__ trans,
                                                                const float* __restrict__ posedirs,
                                                                const float* __restrict__ weights,
                                                                const float* __restrict__ v_base,
                                                                const float* __restrict__ basis,
                                                                const float* __restrict__ frame, float* __restrict__ verts,
                                                                float* __restrict__ verts_cano) {
  const int t = *tptr;
  if (t < 0 || t >= T) return;
  __shared__ SkinShared sh;
  const int n3 = 3 * V, x = threadIdx.x, y = threadIdx.y, tid = y * FL_COLS + x;
  const int c = blockIdx.x * FL_COLS + x;
  float ev[FL_ME], pv[FL_MP];
  load_basis(c, n3, y, NE, basis, posedirs, ev, pv);
  float vs;
  skin_front(sh, t, NE, n3, expr, frame, v_base, ev, pv, &vs);
  if (y == 0 && c < n3 && verts_cano != nullptr) verts_cano[c] = vs;
  const int v = blockIdx.x * FL_TV + tid;
  if (tid < FL_TV && v < V) {
    float w[FL_J], Tv[12];
#pragma unroll
    for (int j = 0; j < FL_J; j++) w[j] = weights[(size_t)v * FL_J + j];
    blend_transform(w, sh.A, Tv);
    const float p0 = sh.vp[3 * tid], p1 = sh.vp[3 * tid + 1], p2 = sh.vp[3 * tid + 2];
#pragma unroll
    for (int r = 0; r < 3; r++)
      verts[3 * (size_t)v + r] = (Tv[4 * r] * p0 + Tv[4 * r + 1] * p1 + Tv[4 * r + 2] * p2 + Tv[4 * r + 3]) + trans[3 * t + r];
  }
}

struct SkinBwdShared {
  float g[FL_TV][3];
  float w[FL_TV][FL_J];
  float vh[FL_TV][4];
  float dvp[FL_COLS];
  float dvs[FL_COLS];
  float red[3][GAB200_FLAME_MAX_EXPR + FL_PB];   // one row per warp of a slice
};

__device__ __forceinline__ float warp_sum(float v) {   // butterfly: every lane ends with the same, fixed-order sum
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct FlameGradPtrs {
  float* g[6];   // expr, rotation, neck, jaw, eyes, translation
};

__global__ void __launch_bounds__(FL_THREADS) flame_skin_backward_kernel(
    int V, int T, int NE, const int32_t* __restrict__ tptr, const float* __restrict__ expr,
    const float* __restrict__ posedirs, const float* __restrict__ weights, const float* __restrict__ v_base,
    const float* __restrict__ basis, const float* __restrict__ frame, const float* __restrict__ g_verts,
    const float* __restrict__ g_cano, float* __restrict__ partials, int pstride, FlameGradPtrs out) {
  const int t = *tptr;
  if (t < 0 || t >= T) return;
  __shared__ SkinShared sh;
  __shared__ SkinBwdShared sb;
  const int n3 = 3 * V, x = threadIdx.x, y = threadIdx.y, tid = y * FL_COLS + x;
  const int c = blockIdx.x * FL_COLS + x;
  // the gradient rows of the other timesteps are exact zeros (row t is written by flame_joints_backward_kernel)
  {
    const int widths[6] = {NE, 3, 3, 3, 6, 3};
    const size_t stride = (size_t)gridDim.x * FL_THREADS, first = (size_t)blockIdx.x * FL_THREADS + tid;
    for (int k = 0; k < 6; k++) {
      const size_t n = (size_t)T * widths[k], lo = (size_t)t * widths[k], hi = lo + widths[k];
      for (size_t i = first; i < n; i += stride)
        if (i < lo || i >= hi) out.g[k][i] = 0.f;
    }
  }
  float ev[FL_ME], pv[FL_MP];
  load_basis(c, n3, y, NE, basis, posedirs, ev, pv);
  float vs;
  skin_front(sh, t, NE, n3, expr, frame, v_base, ev, pv, &vs);
  const int v = blockIdx.x * FL_TV + tid;
  if (tid < FL_TV) {
    float w[FL_J] = {0.f, 0.f, 0.f, 0.f, 0.f}, g[3] = {0.f, 0.f, 0.f}, gc[3] = {0.f, 0.f, 0.f};
    if (v < V) {
#pragma unroll
      for (int j = 0; j < FL_J; j++) w[j] = weights[(size_t)v * FL_J + j];
#pragma unroll
      for (int r = 0; r < 3; r++) {
        g[r] = g_verts[3 * (size_t)v + r];
        if (g_cano != nullptr) gc[r] = g_cano[3 * (size_t)v + r];
      }
    }
    float Tv[12];
    blend_transform(w, sh.A, Tv);
#pragma unroll
    for (int k = 0; k < 3; k++) {   // dv_posed = T_v[:3,:3]^T g
      const float d = Tv[k] * g[0] + Tv[4 + k] * g[1] + Tv[8 + k] * g[2];
      sb.dvp[3 * tid + k] = d;
      sb.dvs[3 * tid + k] = d + gc[k];
      sb.g[tid][k] = g[k];
      sb.vh[tid][k] = v < V ? sh.vp[3 * tid + k] : 0.f;
    }
    sb.vh[tid][3] = v < V ? 1.f : 0.f;
#pragma unroll
    for (int j = 0; j < FL_J; j++) sb.w[tid][j] = w[j];
  }
  __syncthreads();
  // E^T.dv_shaped and P^T.dv_posed over this CTA's 96 coordinates: a warp sum per component, then 3 warps in order
  const float dvs = sb.dvs[x], dvp = sb.dvp[x];
  const int wq = x / 32, lane = x % 32;
#pragma unroll
  for (int i = 0; i < FL_ME; i++) {
    const int e = y + i * FL_S;
    if (e < NE) {   // uniform per warp (a warp lies in one slice)
      const float s = warp_sum(ev[i] * dvs);
      if (lane == 0) sb.red[wq][e] = s;
    }
  }
#pragma unroll
  for (int i = 0; i < FL_MP; i++) {
    const int p = y + i * FL_S;
    if (p < FL_PB) {
      const float s = warp_sum(pv[i] * dvp);
      if (lane == 0) sb.red[wq][GAB200_FLAME_MAX_EXPR + p] = s;
    }
  }
  __syncthreads();
  float* part = partials + (size_t)blockIdx.x * pstride;
  if (tid < 60) {   // dA_j[r][m] = sum_v w_vj g_v[r] [v_posed, 1][m]
    const int j = tid / 12, r = (tid % 12) / 4, m = tid % 4;
    float s = 0.f;
    for (int q = 0; q < FL_TV; q++) s = fmaf(sb.w[q][j] * sb.g[q][r], sb.vh[q][m], s);
    part[FL_P_A + tid] = s;
  } else if (tid < FL_P_TR) {
    const int p = tid - FL_P_PF;
    part[tid] = (sb.red[0][GAB200_FLAME_MAX_EXPR + p] + sb.red[1][GAB200_FLAME_MAX_EXPR + p]) +
                sb.red[2][GAB200_FLAME_MAX_EXPR + p];
  } else if (tid < FL_P_EX) {
    const int r = tid - FL_P_TR;
    float s = 0.f;
    for (int q = 0; q < FL_TV; q++) s += sb.g[q][r];
    part[tid] = s;
  } else if (tid < FL_P_EX + NE) {
    const int e = tid - FL_P_EX;
    part[tid] = (sb.red[0][e] + sb.red[1][e]) + sb.red[2][e];
  }
}

__global__ void __launch_bounds__(256) flame_joints_backward_kernel(
    int T, int NE, FlameParents par, const int32_t* __restrict__ tptr, const float* __restrict__ expr,
    const float* __restrict__ rot, const float* __restrict__ neck, const float* __restrict__ jaw,
    const float* __restrict__ eyes, const float* __restrict__ J_base, const float* __restrict__ JS,
    const float* __restrict__ partials, int n_blocks, int pstride, FlameGradPtrs out) {
  const int t = *tptr;
  if (t < 0 || t >= T) return;
  __shared__ double sum[FL_P_EX + GAB200_FLAME_MAX_EXPR];
  __shared__ double sJ[15], dJ[15], dpose[15];
  const int tid = threadIdx.x;
  for (int k = tid; k < FL_P_EX + NE; k += blockDim.x) {   // CTA order: bit-identical on every call
    double s = 0.0;
    for (int b = 0; b < n_blocks; b++) s += (double)partials[(size_t)b * pstride + k];
    sum[k] = s;
  }
  if (tid < 15) {
    const float* js = JS + (size_t)tid * NE;
    const float* ex = expr + (size_t)t * NE;
    double acc = J_base[tid];
    for (int e = 0; e < NE; e++) acc += (double)js[e] * (double)ex[e];
    sJ[tid] = acc;
  }
  __syncthreads();
  __shared__ Chain ch;   // single-thread work: shared memory keeps the double arrays out of registers and local memory
  __shared__ ChainGrad cg;
  if (tid == 0) {
    for (int i = 0; i < 15; i++) ch.J[i / 3][i % 3] = sJ[i];
    load_pose(t, rot, neck, jaw, eyes, ch.pose);
    chain_forward(ch, par);
    double(&dRc)[FL_J][9] = cg.dRc;
    double(&dtc)[FL_J][3] = cg.dtc;
    double(&dR)[FL_J][9] = cg.dR;
    double(&drel)[FL_J][3] = cg.drel;
    double(&gJ)[FL_J][3] = cg.gJ;
#pragma unroll 1
    for (int i = 0; i < FL_J; i++) {
      // A_i = [Rc | tc - Rc J_i]
      const double* G = sum + FL_P_A + 12 * i;
      for (int r = 0; r < 3; r++) {
        dtc[i][r] = G[4 * r + 3];
        for (int k = 0; k < 3; k++) dRc[i][3 * r + k] = G[4 * r + k] - G[4 * r + 3] * ch.J[i][k];
      }
      for (int k = 0; k < 3; k++)
        gJ[i][k] = -(ch.Rc[i][k] * G[3] + ch.Rc[i][3 + k] * G[7] + ch.Rc[i][6 + k] * G[11]);
      for (int m = 0; m < 9; m++) dR[i][m] = i > 0 ? sum[FL_P_PF + 9 * (i - 1) + m] : 0.0;
    }
#pragma unroll 1
    for (int i = FL_J - 1; i >= 1; i--) {   // children before parents (parents[i] < i)
      const int p = par.p[i];
      const double* Rp = ch.Rc[p];
      const double* Ri = ch.rod[i].R;
      for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) {   // Rc_i = Rp Ri,  tc_i = Rp rel_i + tp
          dRc[p][3 * r + c] += dRc[i][3 * r] * Ri[3 * c] + dRc[i][3 * r + 1] * Ri[3 * c + 1] +
                               dRc[i][3 * r + 2] * Ri[3 * c + 2] + dtc[i][r] * ch.rel[i][c];
          dR[i][3 * r + c] += Rp[r] * dRc[i][c] + Rp[3 + r] * dRc[i][3 + c] + Rp[6 + r] * dRc[i][6 + c];
        }
        dtc[p][r] += dtc[i][r];
        drel[i][r] = Rp[r] * dtc[i][0] + Rp[3 + r] * dtc[i][1] + Rp[6 + r] * dtc[i][2];
      }
    }
    for (int m = 0; m < 9; m++) dR[0][m] += dRc[0][m];
    for (int k = 0; k < 3; k++) drel[0][k] = dtc[0][k];
    for (int k = 0; k < 3; k++) gJ[0][k] += drel[0][k];
    for (int i = 1; i < FL_J; i++)
      for (int k = 0; k < 3; k++) {
        gJ[i][k] += drel[i][k];
        gJ[par.p[i]][k] -= drel[i][k];
      }
#pragma unroll 1
    for (int i = 0; i < FL_J; i++) {
      double dr[3];
      rodrigues_backward(ch.pose + 3 * i, ch.rod[i], dR[i], dr);
      for (int k = 0; k < 3; k++) {
        dpose[3 * i + k] = dr[k];
        dJ[3 * i + k] = gJ[i][k];
      }
    }
  }
  __syncthreads();
  if (tid < NE) {
    double s = sum[FL_P_EX + tid];
    for (int k = 0; k < 15; k++) s += (double)JS[(size_t)k * NE + tid] * dJ[k];
    out.g[0][(size_t)t * NE + tid] = (float)s;
  } else if (tid >= 128 && tid < 128 + 15) {
    const int k = tid - 128;
    if (k < 3) out.g[1][3 * t + k] = (float)dpose[k];
    else if (k < 6) out.g[2][3 * t + k - 3] = (float)dpose[k];
    else if (k < 9) out.g[3][3 * t + k - 6] = (float)dpose[k];
    else out.g[4][6 * t + k - 9] = (float)dpose[k];
  } else if (tid >= 160 && tid < 163) {
    out.g[5][3 * t + tid - 160] = (float)sum[FL_P_TR + tid - 160];
  }
}

// ---- launches -----------------------------------------------------------------------------------------------------
static FlameParents parents_of(const gab200_flame_assets& a) {
  FlameParents p;
  for (int i = 0; i < FL_J; i++) p.p[i] = a.parents[i];
  return p;
}

void launch_flame_prepare(const gab200_flame_assets& a, const float* shape, const float* static_offset, void* scratch,
                          cudaStream_t stream) {
  FlameView f = carve_flame(scratch, a.V, a.n_expr);
  const int n3 = 3 * a.V;
  flame_prepare_vertex_kernel<<<(n3 + 255) / 256, 256, 0, stream>>>(a.V, a.n_shape, a.n_expr, a.v_template, a.shapedirs,
                                                                    shape, static_offset, f.v_base, f.basis);
  count_launch();
  flame_prepare_joint_kernel<<<dim3(15, 1 + a.n_expr), 256, 0, stream>>>(a.V, a.n_expr, a.J_regressor, f.v_base, f.basis,
                                                                         f.J_base, f.JS);
  count_launch();
}

void launch_flame_forward(const gab200_flame_frame_args& g, float* verts, float* verts_cano, cudaStream_t stream) {
  const gab200_flame_assets& a = *g.assets;
  FlameView f = carve_flame(const_cast<void*>(g.scratch), a.V, a.n_expr);
  flame_joints_kernel<<<1, 32, 0, stream>>>(g.T, a.n_expr, parents_of(a), g.timestep, g.expr, g.rotation, g.neck_pose,
                                            g.jaw_pose, g.eyes_pose, g.translation, f.J_base, f.JS, g.frame);
  count_launch();
  flame_skin_kernel<<<f.n_blocks, dim3(FL_COLS, FL_S), 0, stream>>>(a.V, g.T, a.n_expr, g.timestep, g.expr,
                                                                    g.translation, a.posedirs, a.lbs_weights, f.v_base,
                                                                    f.basis, g.frame, verts, verts_cano);
  count_launch();
}

void launch_flame_backward(const gab200_flame_frame_args& g, const float* g_verts, const float* g_cano,
                           const gab200_flame_grads& gr, cudaStream_t stream) {
  const gab200_flame_assets& a = *g.assets;
  FlameView f = carve_flame(const_cast<void*>(g.scratch), a.V, a.n_expr);
  FlameGradPtrs out = {{gr.expr, gr.rotation, gr.neck_pose, gr.jaw_pose, gr.eyes_pose, gr.translation}};
  flame_skin_backward_kernel<<<f.n_blocks, dim3(FL_COLS, FL_S), 0, stream>>>(
      a.V, g.T, a.n_expr, g.timestep, g.expr, a.posedirs, a.lbs_weights, f.v_base, f.basis, g.frame, g_verts, g_cano,
      f.partials, f.pstride, out);
  count_launch();
  flame_joints_backward_kernel<<<1, 256, 0, stream>>>(g.T, a.n_expr, parents_of(a), g.timestep, g.expr, g.rotation,
                                                      g.neck_pose, g.jaw_pose, g.eyes_pose, f.J_base, f.JS, f.partials,
                                                      f.n_blocks, f.pstride, out);
  count_launch();
}

}  // namespace gab
