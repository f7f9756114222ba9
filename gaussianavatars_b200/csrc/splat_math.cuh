// splat_math.cuh -- device math shared by preprocess.cu (compiled --fmad=false, bit-reproducible) and
// preprocess_bwd.cu (default contraction).  Each translation unit gets its own copy under its own flags.
#pragma once
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

#define PRE_NT 64                  // threads per block of the per-splat kernels
#define SH_SMEM_STRIDE_MAX 49      // 16 coefficients * 3 channels, padded to an odd stride

// Cooperative copy of rows [row0, row0+rows) of a row-major [*, width] float matrix into shared memory with row
// stride `pstride` (odd -> the later per-thread row reads are bank-conflict free).  Global side: 128-bit loads.
template <int NT>
__device__ __forceinline__ void stage_rows_in(float* smem, const float* __restrict__ g, size_t row0, int rows, int width,
                                              int pstride) {
  const float* src = g + row0 * (size_t)width;
  const int total = rows * width;
  const int nvec = ((reinterpret_cast<uintptr_t>(src) & 15) == 0) ? total / 4 : 0;
  for (int v = threadIdx.x; v < nvec; v += NT) {
    const float4 x = __ldg(reinterpret_cast<const float4*>(src) + v);
    const int g0 = 4 * v;
    int r = g0 / width, e = g0 - r * width;
    const float vals[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
      smem[r * pstride + e] = vals[k];
      if (++e == width) { e = 0; ++r; }
    }
  }
  for (int q = nvec * 4 + threadIdx.x; q < total; q += NT) {
    const int r = q / width;
    smem[r * pstride + (q - r * width)] = src[q];
  }
}
// NVLS multicast reduction: adds into the same offset of every rank's replica of a symmetric buffer (sm_90+).
__device__ __forceinline__ void mc_red_add(float* mc_addr, float v) {
  asm volatile("multimem.red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(mc_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void mc_red_add4(float* mc_addr, float4 v) {
  asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_addr), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}
template <bool MC>
__device__ __forceinline__ void put(float* addr, float v) {
  if (MC) mc_red_add(addr, v);
  else *addr = v;
}

// The reverse: rows staged in shared memory -> global, 128-bit stores (MC: 128-bit multicast reductions).
template <int NT, bool MC = false>
__device__ __forceinline__ void stage_rows_out(const float* smem, float* __restrict__ g, size_t row0, int rows,
                                               int width, int pstride) {
  float* dst = g + row0 * (size_t)width;
  const int total = rows * width;
  const int nvec = ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) ? total / 4 : 0;
  for (int v = threadIdx.x; v < nvec; v += NT) {
    const int g0 = 4 * v;
    int r = g0 / width, e = g0 - r * width;
    float vals[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      vals[k] = smem[r * pstride + e];
      if (++e == width) { e = 0; ++r; }
    }
    const float4 o = make_float4(vals[0], vals[1], vals[2], vals[3]);
    if (MC) {
      if (o.x != 0.f || o.y != 0.f || o.z != 0.f || o.w != 0.f) mc_red_add4(dst + 4 * (size_t)v, o);
    } else {
      reinterpret_cast<float4*>(dst)[v] = o;
    }
  }
  for (int q = nvec * 4 + threadIdx.x; q < total; q += NT) {
    const int r = q / width;
    put<MC>(dst + q, smem[r * pstride + (q - r * width)]);
  }
}

// Where a per-splat kernel's camera comes from:
//   CAM_ARGS   : the by-value matrices and tanfovx / tanfovy of `a` (gab200_forward, gab200_backward).
//   CAM_DEVFOV : the same matrices, (tanfovx, tanfovy) from a device float[2] `tanfov` (gab200_forward_device_fov,
//                gab200_backward_device_fov), so that a captured graph runs whatever field of view was written before
//                the replay.
//   CAM_TABLE  : rows of the device camera table (the *_views* forms), each row's field of view read as CAM_DEVFOV
//                reads it.
enum { CAM_ARGS, CAM_DEVFOV, CAM_TABLE };

// the camera of a block: viewmatrix (16) | projmatrix (16) | campos (3)
__device__ __forceinline__ void stage_camera(const float* __restrict__ V, const float* __restrict__ Pm,
                                             const float* __restrict__ campos, Camera& cam) {
  int t = threadIdx.x;
  if (t < 16) cam.V[t] = V[t];
  else if (t < 32) cam.Pm[t - 16] = Pm[t - 16];
  else if (t < 35) cam.campos[t - 32] = campos[t - 32];
  __syncthreads();
}

__device__ __forceinline__ float3 xform4x3(const float* M, float3 p) {
  float3 r;
  r.x = M[0] * p.x + M[4] * p.y + M[8] * p.z + M[12];
  r.y = M[1] * p.x + M[5] * p.y + M[9] * p.z + M[13];
  r.z = M[2] * p.x + M[6] * p.y + M[10] * p.z + M[14];
  return r;
}

__device__ __forceinline__ float ndc2pix(float v, int S) {
  return (float)((((double)v + 1.0) * (double)S - 1.0) * 0.5);
}

__device__ __forceinline__ void tile_rect(float px, float py, int radius, int gx, int gy, int& x0, int& y0, int& x1,
                                          int& y1) {
  x0 = min(gx, max(0, (int)((px - (float)radius) / (float)GAB_TILE)));
  y0 = min(gy, max(0, (int)((py - (float)radius) / (float)GAB_TILE)));
  x1 = min(gx, max(0, (int)((px + (float)radius + (float)(GAB_TILE - 1)) / (float)GAB_TILE)));
  y1 = min(gy, max(0, (int)((py + (float)radius + (float)(GAB_TILE - 1)) / (float)GAB_TILE)));
}

__device__ __forceinline__ void quat_to_R(float r, float x, float y, float z, float R[9]) {
  R[0] = 1.f - 2.f * (y * y + z * z);
  R[1] = 2.f * (x * y - r * z);
  R[2] = 2.f * (x * z + r * y);
  R[3] = 2.f * (x * y + r * z);
  R[4] = 1.f - 2.f * (x * x + z * z);
  R[5] = 2.f * (y * z - r * x);
  R[6] = 2.f * (x * z - r * y);
  R[7] = 2.f * (y * z + r * x);
  R[8] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = R diag(s^2) R^T from a rotation matrix and s (already multiplied by scale_modifier)
__device__ __forceinline__ void cov3d_from_R(const float R[9], const float s[3], float cov[6]) {
  float M[9];
#pragma unroll
  for (int k = 0; k < 3; k++)
#pragma unroll
    for (int i = 0; i < 3; i++) M[3 * k + i] = s[k] * R[3 * i + k];
  cov[0] = M[0] * M[0] + M[3] * M[3] + M[6] * M[6];
  cov[1] = M[0] * M[1] + M[3] * M[4] + M[6] * M[7];
  cov[2] = M[0] * M[2] + M[3] * M[5] + M[6] * M[8];
  cov[3] = M[1] * M[1] + M[4] * M[4] + M[7] * M[7];
  cov[4] = M[1] * M[2] + M[4] * M[5] + M[7] * M[8];
  cov[5] = M[2] * M[2] + M[5] * M[5] + M[8] * M[8];
}

// ---- the binding + activation of scene/gaussian_model.py:113-160, shared by forward / export / backward ----
struct Activated {
  float3 mean;     // world position
  float opacity;   // sigmoid
  float s[3];      // exp(_scaling) * face_scaling          (WITHOUT scale_modifier)
  float R[9];      // world rotation R_face * R(normalize(_rotation))
};
// intermediates the backward chain needs (dead code in the forward instantiation)
struct BindCtx {
  float3 xl;       // raw local position
  float qn[4];     // normalised local quaternion (wxyz)
  float nrm;       // max(|q|, 1e-12)
  float e[3];      // exp(_scaling)
  float fs;        // face scale (1 when unbound)
  float Rf[9];     // face frame (identity when unbound)
  float Rl[9];     // R(qn)
  float3 rx;       // R_face * xl
  int face;        // -1 when unbound
};

// The 11 per-splat floats besides the SH coefficients (position, quaternion, scales, opacity; raw or activated
// depending on the input mode).  The quaternion is one float4 (LDG.128) per thread; positions and scales have a
// 12-byte stride and are read as coalesced scalars: staging them through shared memory for LDG.128 would cost a
// barrier for 24 of the 284 bytes of a splat.
struct RawAttr {
  float x[3], q[4], s[3], o;
};
// 16-byte aligned quaternion array -> one LDG.128 per splat
__device__ __forceinline__ void load_quat(const float* __restrict__ rot, size_t i, float q[4]) {
  if ((reinterpret_cast<uintptr_t>(rot) & 15) == 0) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(rot) + i);
    q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
  } else {
    q[0] = rot[4 * i]; q[1] = rot[4 * i + 1]; q[2] = rot[4 * i + 2]; q[3] = rot[4 * i + 3];
  }
}
// straight from global memory
__device__ __forceinline__ void load_raw(const gab200_forward_args& a, int i, RawAttr& r) {
#pragma unroll
  for (int k = 0; k < 3; k++) r.x[k] = a.means3D[3 * (size_t)i + k];
  if (a.rotations != nullptr) load_quat(a.rotations, (size_t)i, r.q);
  if (a.scales != nullptr) {
#pragma unroll
    for (int k = 0; k < 3; k++) r.s[k] = a.scales[3 * (size_t)i + k];
  }
  r.o = a.opacities[i];
}

__device__ __forceinline__ void bind_activate(const gab200_forward_args& a, int i, const RawAttr& raw, Activated& o,
                                              BindCtx& c) {
  c.xl = make_float3(raw.x[0], raw.x[1], raw.x[2]);
  // rotation_activation = torch.nn.functional.normalize (eps 1e-12)
  float qr = raw.q[0], qx = raw.q[1], qy = raw.q[2], qz = raw.q[3];
  float n = sqrtf(qr * qr + qx * qx + qy * qy + qz * qz);
  n = fmaxf(n, 1e-12f);
  c.nrm = n;
  c.qn[0] = qr / n; c.qn[1] = qx / n; c.qn[2] = qy / n; c.qn[3] = qz / n;
  quat_to_R(c.qn[0], c.qn[1], c.qn[2], c.qn[3], c.Rl);
  c.e[0] = expf(raw.s[0]);
  c.e[1] = expf(raw.s[1]);
  c.e[2] = expf(raw.s[2]);
  o.opacity = 1.0f / (1.0f + expf(-raw.o));
  if (a.binding != nullptr) {
    const int f = a.binding[i];
    c.face = f;
    const float* Rf = a.face_orien_mat + 9 * (size_t)f;
    c.fs = a.face_scaling[f];
    const float* fc = a.face_center + 3 * (size_t)f;
#pragma unroll
    for (int k = 0; k < 9; k++) c.Rf[k] = Rf[k];
    // get_xyz: bmm(R_face, x) * s + c
    c.rx.x = c.Rf[0] * c.xl.x + c.Rf[1] * c.xl.y + c.Rf[2] * c.xl.z;
    c.rx.y = c.Rf[3] * c.xl.x + c.Rf[4] * c.xl.y + c.Rf[5] * c.xl.z;
    c.rx.z = c.Rf[6] * c.xl.x + c.Rf[7] * c.xl.y + c.Rf[8] * c.xl.z;
    o.mean = make_float3(c.rx.x * c.fs + fc[0], c.rx.y * c.fs + fc[1], c.rx.z * c.fs + fc[2]);
    o.s[0] = c.e[0] * c.fs; o.s[1] = c.e[1] * c.fs; o.s[2] = c.e[2] * c.fs;
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int cc = 0; cc < 3; cc++)
        o.R[3 * r + cc] = c.Rf[3 * r + 0] * c.Rl[0 + cc] + c.Rf[3 * r + 1] * c.Rl[3 + cc] + c.Rf[3 * r + 2] * c.Rl[6 + cc];
  } else {
    c.face = -1;
    c.fs = 1.f;
#pragma unroll
    for (int k = 0; k < 9; k++) c.Rf[k] = (k % 4 == 0) ? 1.f : 0.f;
    c.rx = c.xl;
    o.mean = c.xl;
    o.s[0] = c.e[0]; o.s[1] = c.e[1]; o.s[2] = c.e[2];
#pragma unroll
    for (int k = 0; k < 9; k++) o.R[k] = c.Rl[k];
  }
}
__device__ __forceinline__ void bind_activate(const gab200_forward_args& a, int i, Activated& o, BindCtx& c) {
  RawAttr raw;
  load_raw(a, i, raw);
  bind_activate(a, i, raw, o, c);
}
__device__ __forceinline__ void bind_activate(const gab200_forward_args& a, int i, Activated& o) {
  BindCtx c;
  bind_activate(a, i, o, c);
}

__device__ __forceinline__ void sh_basis(int deg, float3 d, float B[16]) {
  B[0] = SH_C0;
  if (deg > 0) {
    float x = d.x, y = d.y, z = d.z;
    B[1] = -SH_C1 * y;
    B[2] = SH_C1 * z;
    B[3] = -SH_C1 * x;
    if (deg > 1) {
      float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
      B[4] = SH_C2_0 * xy;
      B[5] = SH_C2_1 * yz;
      B[6] = SH_C2_2 * (2.0f * zz - xx - yy);
      B[7] = SH_C2_3 * xz;
      B[8] = SH_C2_4 * (xx - yy);
      if (deg > 2) {
        B[9] = SH_C3_0 * y * (3.0f * xx - yy);
        B[10] = SH_C3_1 * xy * z;
        B[11] = SH_C3_2 * y * (4.0f * zz - xx - yy);
        B[12] = SH_C3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
        B[13] = SH_C3_4 * x * (4.0f * zz - xx - yy);
        B[14] = SH_C3_5 * z * (xx - yy);
        B[15] = SH_C3_6 * x * (xx - 3.0f * yy);
      }
    }
  }
}


}  // namespace gab
