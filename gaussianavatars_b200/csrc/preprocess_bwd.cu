// preprocess_bwd.cu -- per-splat backward: 2-D gradients (from blend-backward) -> parameter gradients, with the
// FLAME binding chain fused in.  One kernel replaces computeCov2DCUDA + preprocessCUDA(bwd) of the reference module
// (SURVEY.md 2.4 K8/K9, Appendix B.5) AND the autograd graph of scene/gaussian_model.py:113-160 (SURVEY.md 8a/a15):
// in BOUND_RAW mode it emits dL/d{_xyz, _rotation(raw), _scaling(log), _opacity(logit), f_dc, f_rest} and
// accumulates dL/d{face_center, face_orien_mat, face_scaling}.
// Behavioural quirks of the reference module are kept (Appendix B.5): 1/(det^2+1e-7) guard, guard-band masks,
// no quaternion-normalisation Jacobian in ACTIVATED mode, dL/dscale w.r.t. s = mod*scale without the extra mod.
#include <cstdlib>

#include "common.cuh"
#include "kernels.cuh"
#include "splat_math.cuh"

namespace gab {

// One camera's part of the backward of a splat with mean m and covariance c3: the 2-D gradients of its g2d row `g`
// -> dL/dSigma (gcov) and dL/dmean (gm) through that camera's projection.  DEVFOV: (tanfovx, tanfovy) from the device
// float[2] `tanfov` the forward read.  DA: g slot 9 holds dL/dz of the depth plane, added to gm through the camera's
// t.z = V[2] x + V[6] y + V[10] z + V[14].
template <bool DEVFOV, bool DA>
__device__ __forceinline__ void view_backward(const gab200_forward_args& a, const Camera& cam, const float* tanfov,
                                              float3 m, const float c3[6], const float* g, float gm[3],
                                              float gcov[6]) {
  const int W = a.image_width, H = a.image_height;
  const float g2x = g[0], g2y = g[1], gA = g[2], gB = g[3], gC = g[4];
  // ---- conic -> cov2D -> Sigma, t -> mean ----
  const float* V = cam.V;
  // visible splats only: the forward culled every splat when the device field of view was invalid
  const float tanfovx = DEVFOV ? __ldg(tanfov) : a.tanfovx, tanfovy = DEVFOV ? __ldg(tanfov + 1) : a.tanfovy;
  const float fx = (float)W / (2.0f * tanfovx), fy = (float)H / (2.0f * tanfovy);
  float3 t = xform4x3(V, m);
  const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
  const float txtz = t.x / t.z, tytz = t.y / t.z;
  const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
  const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
  t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
  t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
  const float j00 = fx / t.z, j02 = -(fx * t.x) / (t.z * t.z);
  const float j11 = fy / t.z, j12 = -(fy * t.y) / (t.z * t.z);
  float T0[3], T1[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    T0[c] = j00 * V[4 * c + 0] + j02 * V[4 * c + 2];
    T1[c] = j11 * V[4 * c + 1] + j12 * V[4 * c + 2];
  }
  const float S[9] = {c3[0], c3[1], c3[2], c3[1], c3[3], c3[4], c3[2], c3[4], c3[5]};
  float u[3], v[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
    u[r] = S[3 * r + 0] * T0[0] + S[3 * r + 1] * T0[1] + S[3 * r + 2] * T0[2];
    v[r] = S[3 * r + 0] * T1[0] + S[3 * r + 1] * T1[1] + S[3 * r + 2] * T1[2];
  }
  const float ca = T0[0] * u[0] + T0[1] * u[1] + T0[2] * u[2] + 0.3f;
  const float cb = T0[0] * v[0] + T0[1] * v[1] + T0[2] * v[2];
  const float cc = T1[0] * v[0] + T1[1] * v[1] + T1[2] * v[2] + 0.3f;
  const float denom = ca * cc - cb * cb;
  const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
  float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
#pragma unroll
  for (int k = 0; k < 6; k++) gcov[k] = 0.f;
  if (denom2inv != 0.f) {
    dL_da = denom2inv * (-cc * cc * gA + 2 * cb * cc * gB + (denom - ca * cc) * gC);
    dL_dc = denom2inv * (-ca * ca * gC + 2 * ca * cb * gB + (denom - ca * cc) * gA);
    dL_db = denom2inv * 2 * (cb * cc * gA - (denom + 2 * cb * cb) * gB + ca * cb * gC);
    gcov[0] = T0[0] * T0[0] * dL_da + T0[0] * T1[0] * dL_db + T1[0] * T1[0] * dL_dc;
    gcov[3] = T0[1] * T0[1] * dL_da + T0[1] * T1[1] * dL_db + T1[1] * T1[1] * dL_dc;
    gcov[5] = T0[2] * T0[2] * dL_da + T0[2] * T1[2] * dL_db + T1[2] * T1[2] * dL_dc;
    gcov[1] = 2 * T0[0] * T0[1] * dL_da + (T0[0] * T1[1] + T0[1] * T1[0]) * dL_db + 2 * T1[0] * T1[1] * dL_dc;
    gcov[2] = 2 * T0[0] * T0[2] * dL_da + (T0[0] * T1[2] + T0[2] * T1[0]) * dL_db + 2 * T1[0] * T1[2] * dL_dc;
    gcov[4] = 2 * T0[2] * T0[1] * dL_da + (T0[1] * T1[2] + T0[2] * T1[1]) * dL_db + 2 * T1[1] * T1[2] * dL_dc;
  }
  // u = S T0^T, v = S T1^T  (S symmetric):  dT0 = 2 u dL_da + v dL_db ; dT1 = 2 v dL_dc + u dL_db
  float dT0[3], dT1[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    dT0[k] = 2 * u[k] * dL_da + v[k] * dL_db;
    dT1[k] = 2 * v[k] * dL_dc + u[k] * dL_db;
  }
  const float dJ00 = V[0] * dT0[0] + V[4] * dT0[1] + V[8] * dT0[2];
  const float dJ02 = V[2] * dT0[0] + V[6] * dT0[1] + V[10] * dT0[2];
  const float dJ11 = V[1] * dT1[0] + V[5] * dT1[1] + V[9] * dT1[2];
  const float dJ12 = V[2] * dT1[0] + V[6] * dT1[1] + V[10] * dT1[2];
  const float tz = 1.f / t.z, tz2 = tz * tz, tz3 = tz2 * tz;
  const float dtx = x_grad_mul * -fx * tz2 * dJ02;
  const float dty = y_grad_mul * -fy * tz2 * dJ12;
  const float dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + (2 * fx * t.x) * tz3 * dJ02 + (2 * fy * t.y) * tz3 * dJ12;
#pragma unroll
  for (int k = 0; k < 3; k++) gm[k] = V[4 * k + 0] * dtx + V[4 * k + 1] * dty + V[4 * k + 2] * dtz;

  // ---- projection of the mean ----
  const float* Pm = cam.Pm;
  const float h0 = Pm[0] * m.x + Pm[4] * m.y + Pm[8] * m.z + Pm[12];
  const float h1 = Pm[1] * m.x + Pm[5] * m.y + Pm[9] * m.z + Pm[13];
  const float h3 = Pm[3] * m.x + Pm[7] * m.y + Pm[11] * m.z + Pm[15];
  const float m_w = 1.0f / (h3 + 0.0000001f);
  const float mul1 = h0 * m_w * m_w, mul2 = h1 * m_w * m_w;
  gm[0] += (Pm[0] * m_w - Pm[3] * mul1) * g2x + (Pm[1] * m_w - Pm[3] * mul2) * g2y;
  gm[1] += (Pm[4] * m_w - Pm[7] * mul1) * g2x + (Pm[5] * m_w - Pm[7] * mul2) * g2y;
  gm[2] += (Pm[8] * m_w - Pm[11] * mul1) * g2x + (Pm[9] * m_w - Pm[11] * mul2) * g2y;
  if (DA) {
    const float gz = g[9];
    gm[0] += V[2] * gz;
    gm[1] += V[6] * gz;
    gm[2] += V[10] * gz;
  }
}

// The view-direction term of the SH colour: fills the basis B of the direction from the camera centre `campos` to
// the mean m and adds dL/dcolour (gRGB) through the direction to gm.  my_sh: the splat's staged SH coefficients
// (BOUND: f_rest, coefficient k in row k - 1).
template <bool BOUND>
__device__ __forceinline__ void sh_dir_backward(int sh_degree, const float campos[3], float3 m, const float* my_sh,
                                                const float gRGB[3], float B[16], float gm[3]) {
  const float3 d0 = make_float3(m.x - campos[0], m.y - campos[1], m.z - campos[2]);
  const float s2 = d0.x * d0.x + d0.y * d0.y + d0.z * d0.z;
  const float len = sqrtf(s2);
  const float3 d = make_float3(d0.x / len, d0.y / len, d0.z / len);
  sh_basis(sh_degree, d, B);
  const float x = d.x, y = d.y, z = d.z;
  float gd[3] = {0.f, 0.f, 0.f};
  if (sh_degree > 0) {
    auto SHV = [&](int k, int ch) -> float { return BOUND ? my_sh[3 * (k - 1) + ch] : my_sh[3 * k + ch]; };
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      float dxc = -SH_C1 * SHV(3, ch), dyc = -SH_C1 * SHV(1, ch), dzc = SH_C1 * SHV(2, ch);
      if (sh_degree > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        dxc += SH_C2_0 * y * SHV(4, ch) + SH_C2_2 * 2.f * -x * SHV(6, ch) + SH_C2_3 * z * SHV(7, ch) +
               SH_C2_4 * 2.f * x * SHV(8, ch);
        dyc += SH_C2_0 * x * SHV(4, ch) + SH_C2_1 * z * SHV(5, ch) + SH_C2_2 * 2.f * -y * SHV(6, ch) +
               SH_C2_4 * 2.f * -y * SHV(8, ch);
        dzc += SH_C2_1 * y * SHV(5, ch) + SH_C2_2 * 2.f * 2.f * z * SHV(6, ch) + SH_C2_3 * x * SHV(7, ch);
        if (sh_degree > 2) {
          dxc += SH_C3_0 * SHV(9, ch) * 3.f * 2.f * xy + SH_C3_1 * SHV(10, ch) * yz +
                 SH_C3_2 * SHV(11, ch) * -2.f * xy + SH_C3_3 * SHV(12, ch) * -3.f * 2.f * xz +
                 SH_C3_4 * SHV(13, ch) * (-3.f * xx + 4.f * zz - yy) + SH_C3_5 * SHV(14, ch) * 2.f * xz +
                 SH_C3_6 * SHV(15, ch) * 3.f * (xx - yy);
          dyc += SH_C3_0 * SHV(9, ch) * 3.f * (xx - yy) + SH_C3_1 * SHV(10, ch) * xz +
                 SH_C3_2 * SHV(11, ch) * (-3.f * yy + 4.f * zz - xx) + SH_C3_3 * SHV(12, ch) * -3.f * 2.f * yz +
                 SH_C3_4 * SHV(13, ch) * -2.f * xy + SH_C3_5 * SHV(14, ch) * -2.f * yz +
                 SH_C3_6 * SHV(15, ch) * -3.f * 2.f * xy;
          dzc += SH_C3_1 * SHV(10, ch) * xy + SH_C3_2 * SHV(11, ch) * 4.f * 2.f * yz +
                 SH_C3_3 * SHV(12, ch) * 3.f * (2.f * zz - xx - yy) + SH_C3_4 * SHV(13, ch) * 4.f * 2.f * xz +
                 SH_C3_5 * SHV(14, ch) * (xx - yy);
        }
      }
      gd[0] += dxc * gRGB[ch];
      gd[1] += dyc * gRGB[ch];
      gd[2] += dzc * gRGB[ch];
    }
    const float inv3 = 1.0f / (s2 * len);
    gm[0] += ((s2 - d0.x * d0.x) * gd[0] - d0.y * d0.x * gd[1] - d0.z * d0.x * gd[2]) * inv3;
    gm[1] += (-d0.x * d0.y * gd[0] + (s2 - d0.y * d0.y) * gd[1] - d0.z * d0.y * gd[2]) * inv3;
    gm[2] += (-d0.x * d0.z * gd[0] - d0.y * d0.z * gd[1] + (s2 - d0.z * d0.z) * gd[2]) * inv3;
  }
}

// dL/dSigma (gcov) and dL/dmean (gm) of splat i -> gscale, grot [BOUND: -> the binding chain, the face frame and the
// sigmoid: g_xyz, g_opacity_out].  Rw, s: the world rotation and s = mod * scale the covariance was formed from.
// Every step is linear in gcov, gm and g_op.  The 13 face-frame values go to the splat's row my_fg of the block's
// tile when csr, else into b's face gradients with atomics.
template <bool BOUND>
__device__ __forceinline__ void chain_backward(const gab200_forward_args& a, const gab200_backward_args& b, int i,
                                               const float gcov[6], const float gm[3], float g_op, const float Rw[9],
                                               const float s[3], const Activated& act, const BindCtx& ctx, bool csr,
                                               float* my_fg, float gscale[3], float grot[4], float g_xyz[3],
                                               float& g_opacity_out) {
  const float dS[9] = {gcov[0],        0.5f * gcov[1], 0.5f * gcov[2], 0.5f * gcov[1], gcov[3],
                       0.5f * gcov[4], 0.5f * gcov[2], 0.5f * gcov[4], gcov[5]};
  float A[9], dR[9];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int k = 0; k < 3; k++) A[3 * r + k] = dS[3 * r + 0] * Rw[0 + k] + dS[3 * r + 1] * Rw[3 + k] + dS[3 * r + 2] * Rw[6 + k];
  float gs_in[3];  // gradient w.r.t. the scale fed to the covariance (s / mod), reference convention
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float dot = Rw[0 + k] * A[0 + k] + Rw[3 + k] * A[3 + k] + Rw[6 + k] * A[6 + k];
    gs_in[k] = 2.f * s[k] * dot;
#pragma unroll
    for (int r = 0; r < 3; r++) dR[3 * r + k] = 2.f * s[k] * s[k] * A[3 * r + k];
  }
  float qr, qx, qy, qz;
  float dRl[9];
  if (BOUND) {
    qr = ctx.qn[0]; qx = ctx.qn[1]; qy = ctx.qn[2]; qz = ctx.qn[3];
    // R_w = R_f R_l :  dR_l = R_f^T dR_w ;  dR_f += dR_w R_l^T
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int c = 0; c < 3; c++)
        dRl[3 * r + c] = ctx.Rf[0 + r] * dR[0 + c] + ctx.Rf[3 + r] * dR[3 + c] + ctx.Rf[6 + r] * dR[6 + c];
  } else {
    qr = a.rotations[4 * (size_t)i]; qx = a.rotations[4 * (size_t)i + 1];
    qy = a.rotations[4 * (size_t)i + 2]; qz = a.rotations[4 * (size_t)i + 3];
#pragma unroll
    for (int k = 0; k < 9; k++) dRl[k] = dR[k];
  }
  float gq[4];
  gq[0] = 2.f * (-qz * dRl[1] + qy * dRl[2] + qz * dRl[3] - qx * dRl[5] - qy * dRl[6] + qx * dRl[7]);
  gq[1] = 2.f * (qy * dRl[1] + qz * dRl[2] + qy * dRl[3] - 2.f * qx * dRl[4] - qr * dRl[5] + qz * dRl[6] +
                 qr * dRl[7] - 2.f * qx * dRl[8]);
  gq[2] = 2.f * (-2.f * qy * dRl[0] + qx * dRl[1] + qr * dRl[2] + qx * dRl[3] + qz * dRl[5] - qr * dRl[6] +
                 qz * dRl[7] - 2.f * qy * dRl[8]);
  gq[3] = 2.f * (-2.f * qz * dRl[0] - qr * dRl[1] + qx * dRl[2] + qr * dRl[3] - 2.f * qz * dRl[4] + qy * dRl[5] +
                 qx * dRl[6] + qy * dRl[7]);
  if (BOUND) {
    // through q_n = q / max(|q|, eps)
    const float dotq = qr * gq[0] + qx * gq[1] + qy * gq[2] + qz * gq[3];
    const float inv = 1.f / ctx.nrm;
    grot[0] = (gq[0] - qr * dotq) * inv;
    grot[1] = (gq[1] - qx * dotq) * inv;
    grot[2] = (gq[2] - qy * dotq) * inv;
    grot[3] = (gq[3] - qz * dotq) * inv;
    // s_in = e * fs  ->  log-scale and face scale
    float g_fs = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      gscale[k] = gs_in[k] * ctx.e[k] * ctx.fs;
      g_fs += gs_in[k] * ctx.e[k];
    }
    // mean = fs * (R_f x) + c
    g_xyz[0] = ctx.fs * (ctx.Rf[0] * gm[0] + ctx.Rf[3] * gm[1] + ctx.Rf[6] * gm[2]);
    g_xyz[1] = ctx.fs * (ctx.Rf[1] * gm[0] + ctx.Rf[4] * gm[1] + ctx.Rf[7] * gm[2]);
    g_xyz[2] = ctx.fs * (ctx.Rf[2] * gm[0] + ctx.Rf[5] * gm[1] + ctx.Rf[8] * gm[2]);
    g_opacity_out = g_op * act.opacity * (1.f - act.opacity);
    if (ctx.face >= 0 && csr) {
      // CSR route: leave the 13 contributions in the block's tile; face_grad_reduce_kernel sums them per face
      g_fs += gm[0] * ctx.rx.x + gm[1] * ctx.rx.y + gm[2] * ctx.rx.z;
      my_fg[0] = gm[0]; my_fg[1] = gm[1]; my_fg[2] = gm[2];
      const float xl[3] = {ctx.xl.x, ctx.xl.y, ctx.xl.z};
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++)
          my_fg[3 + 3 * r + c] = dR[3 * r + 0] * ctx.Rl[3 * c + 0] + dR[3 * r + 1] * ctx.Rl[3 * c + 1] +
                                 dR[3 * r + 2] * ctx.Rl[3 * c + 2] + ctx.fs * gm[r] * xl[c];
      my_fg[12] = g_fs;
    } else if (ctx.face >= 0) {
      g_fs += gm[0] * ctx.rx.x + gm[1] * ctx.rx.y + gm[2] * ctx.rx.z;
      const size_t f = (size_t)ctx.face;
      if (b.dL_dface_center != nullptr) {
        atomicAdd(b.dL_dface_center + 3 * f + 0, gm[0]);
        atomicAdd(b.dL_dface_center + 3 * f + 1, gm[1]);
        atomicAdd(b.dL_dface_center + 3 * f + 2, gm[2]);
      }
      if (b.dL_dface_scaling != nullptr) atomicAdd(b.dL_dface_scaling + f, g_fs);
      if (b.dL_dface_orien_mat != nullptr) {
        const float xl[3] = {ctx.xl.x, ctx.xl.y, ctx.xl.z};
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
          for (int c = 0; c < 3; c++) {
            const float viaR = dR[3 * r + 0] * ctx.Rl[3 * c + 0] + dR[3 * r + 1] * ctx.Rl[3 * c + 1] +
                               dR[3 * r + 2] * ctx.Rl[3 * c + 2];
            atomicAdd(b.dL_dface_orien_mat + 9 * f + 3 * r + c, viaR + ctx.fs * gm[r] * xl[c]);
          }
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < 3; k++) gscale[k] = gs_in[k];
#pragma unroll
    for (int k = 0; k < 4; k++) grot[k] = gq[k];
  }
}

// The per-splat backward, one thread per (real) splat.  CAM (splat_math.cuh) says where the camera comes from.
// One camera (CAM_ARGS, CAM_DEVFOV): either input mode; MC: the gradients leave as multimem.red.add (BOUND_RAW only).
// CAM_TABLE (gab200_backward_views*, BOUND_RAW): thread i walks the views in order.  Per view k it stages camera row
//   k, reads the 2-D gradients, radius and clamp bits of virtual splat k * P + i, writes dL/dmeans2D row (k, i) and adds
//   that view's dL/dSigma, dL/dmean (direction term of the SH colour included), dL/dopacity and SH gradients to sums
//   kept in registers (SH: a second shared-memory tile beside the staged coefficients).  Every step after those is
//   linear in them, so the binding chain and the face-frame gradients run once, on the sums, and every gradient is
//   stored once: no cross-view atomics and no per-view gradient scratch.  The binding, the parameter loads and the
//   staged SH rows serve all views.  A view in which the splat is not visible (radius 0 -- also every splat of a view
//   whose tan(FoV/2) is invalid) adds nothing.
// DA: g2d slot 9 of each (virtual) splat holds dL/dz of the depth plane (gab200_backward*_depth_alpha), added to that
//   view's dL/dmean through its own view-matrix row before the chain.  Plain stores only.
// Occupancy: 12 CTAs per SM for the plain one-camera forms (80 registers; the BOUND_RAW ones spill), 8 for the depth
// forms (up to 128 registers: under the 12 their BOUND_RAW instances spill), no minimum for CAM_TABLE.
template <bool BOUND, bool MC, int CAM, bool DA>
__global__ void __launch_bounds__(PRE_NT, CAM == CAM_TABLE ? 0 : DA ? 8 : 12) preprocess_backward_kernel(
    gab200_backward_args b, gab200_forward_args a, int views, const float* __restrict__ cameras,
    const float* __restrict__ tanfov, const SplatAux* __restrict__ aux, const uint8_t* __restrict__ clamped,
    const float* __restrict__ g2d, float* __restrict__ face_scratch) {
  constexpr bool VIEWS = CAM == CAM_TABLE;
  __shared__ Camera cam;
  __shared__ float fg_s[PRE_NT * GAB_FACE_GRAD_STRIDE];  // per-splat face-frame gradients, written out coalesced
  // SH coefficients in (for the view-direction term): coalesced 128-bit global accesses, conflict-free (odd stride)
  // per-thread row accesses.  One camera: the SH gradients go out through the same tile; CAM_TABLE sums them over
  // the views in a second one.
  __shared__ float sh_s[PRE_NT * SH_SMEM_STRIDE_MAX];
  __shared__ float shg_s[VIEWS ? PRE_NT * SH_SMEM_STRIDE_MAX : 1];
  float* my_fg = fg_s + threadIdx.x * GAB_FACE_GRAD_STRIDE;
  if (BOUND && face_scratch != nullptr) {
#pragma unroll
    for (int k = 0; k < GAB_FACE_GRAD_STRIDE; k++) my_fg[k] = 0.f;
  }
  const int M = a.sh_coeffs;
  const int sh_width = BOUND ? 3 * (M - 1) : 3 * M;
  const int sh_stride = sh_width | 1;
  float* my_sh = sh_s + threadIdx.x * sh_stride;
  float* my_shg = VIEWS ? shg_s + threadIdx.x * sh_stride : my_sh;
  if (VIEWS)
    for (int k = 0; k < sh_width; k++) my_shg[k] = 0.f;
  pdl_wait();  // shared-memory set-up above overlaps the predecessor (launch_pdl)
  pdl_trigger();
  if (BOUND && face_scratch != nullptr) {  // face_grad_reduce_kernel adds into the face gradients after this grid
    const size_t F = (size_t)a.num_faces, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < 13 * F; j += stride) {
      float* dst = j < F ? b.dL_dface_scaling : (j < 4 * F ? b.dL_dface_center : b.dL_dface_orien_mat);
      if (dst != nullptr) dst[j < F ? j : (j < 4 * F ? j - F : j - 4 * F)] = 0.f;
    }
  }
  if (!VIEWS) stage_camera(a.viewmatrix, a.projmatrix, a.campos, cam);
  const int row0 = blockIdx.x * PRE_NT;
  const int rows = min(PRE_NT, a.P - row0);
  const float* sh_src = BOUND ? a.sh_rest : a.shs;
  const bool use_sh = (a.colors_precomp == nullptr);
  const bool stage_sh = use_sh && sh_src != nullptr && sh_width > 0;
  if (stage_sh) {
    if (a.sh_degree > 0) stage_rows_in<PRE_NT>(sh_s, sh_src, (size_t)row0, rows, sh_width, sh_stride);
    if (!VIEWS) __syncthreads();  // CAM_TABLE: the barrier before the first view's camera
  }
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = idx < a.P;
  const int i = active ? idx : a.P - 1;
  const int nb = (a.sh_degree + 1) * (a.sh_degree + 1);

  // one camera: this view's gradients; CAM_TABLE: their sums over the views
  float gm[3] = {0.f, 0.f, 0.f}, gcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float gscale[3] = {0.f, 0.f, 0.f}, grot[4] = {0.f, 0.f, 0.f, 0.f};
  float g_op = 0.f, g2x = 0.f, g2y = 0.f, gcol[3] = {0.f, 0.f, 0.f}, gdc[3] = {0.f, 0.f, 0.f};
  bool visible;  // CAM_TABLE: in at least one view

  Activated act;
  BindCtx ctx;
  float3 m;
  float c3[6];
  float Rw[9], s[3];  // world rotation and s = mod * scale (when computed from scale/rotation)
  const bool from_sr = BOUND || (a.cov3D_precomp == nullptr);

  if constexpr (VIEWS) {
    visible = false;
    bind_activate(a, i, act, ctx);
    m = act.mean;
#pragma unroll
    for (int k = 0; k < 9; k++) Rw[k] = act.R[k];
#pragma unroll
    for (int k = 0; k < 3; k++) s[k] = a.scale_modifier * act.s[k];
    cov3d_from_R(Rw, s, c3);
    for (int view = 0; view < views; view++) {
      const float* row = cameras + (size_t)view * GAB200_CAMERA_FLOATS;
      __syncthreads();  // the previous view's camera is no longer read (first view: the SH rows are staged)
      stage_camera(row, row + 16, row + 32, cam);
      const size_t vi = (size_t)view * a.P + i;
      const bool seen = active && aux[vi].radius > 0;
      float vg2x = 0.f, vg2y = 0.f;
      if (seen) {
        visible = true;
        const float* g = g2d + vi * GAB_G2D_STRIDE;
        vg2x = g[0]; vg2y = g[1];
        g_op += g[5];
        const float vgcol[3] = {g[6], g[7], g[8]};
        float vgm[3], vgcov[6];
        view_backward<true, DA>(a, cam, row + 35, m, c3, g, vgm, vgcov);
        if (use_sh) {
          float gRGB[3];
          float B[16];
#pragma unroll
          for (int k = 0; k < 16; k++) B[k] = 0.f;
          const uint8_t cl = clamped[vi];
#pragma unroll
          for (int ch = 0; ch < 3; ch++) gRGB[ch] = ((cl >> ch) & 1) ? 0.f : vgcol[ch];
          sh_dir_backward<BOUND>(a.sh_degree, cam.campos, m, my_sh, gRGB, B, vgm);
#pragma unroll
          for (int ch = 0; ch < 3; ch++) gdc[ch] += B[0] * gRGB[ch];
          for (int k = 1; k < nb && k < M; k++) {
            my_shg[3 * (k - 1) + 0] += B[k] * gRGB[0];
            my_shg[3 * (k - 1) + 1] += B[k] * gRGB[1];
            my_shg[3 * (k - 1) + 2] += B[k] * gRGB[2];
          }
        }
#pragma unroll
        for (int k = 0; k < 3; k++) gm[k] += vgm[k];
#pragma unroll
        for (int k = 0; k < 6; k++) gcov[k] += vgcov[k];
      }
      if (active && b.dL_dmeans2D != nullptr) {
        b.dL_dmeans2D[3 * vi + 0] = vg2x;
        b.dL_dmeans2D[3 * vi + 1] = vg2y;
        b.dL_dmeans2D[3 * vi + 2] = 0.f;
      }
    }
  } else {
    visible = active && aux[i].radius > 0;
    if (visible) {
      const float* g = g2d + (size_t)i * GAB_G2D_STRIDE;
      g2x = g[0]; g2y = g[1];
      g_op = g[5];
      gcol[0] = g[6]; gcol[1] = g[7]; gcol[2] = g[8];

      if (BOUND) {
        bind_activate(a, i, act, ctx);
        m = act.mean;
#pragma unroll
        for (int k = 0; k < 9; k++) Rw[k] = act.R[k];
#pragma unroll
        for (int k = 0; k < 3; k++) s[k] = a.scale_modifier * act.s[k];
        cov3d_from_R(Rw, s, c3);
      } else {
        m = make_float3(a.means3D[3 * (size_t)i], a.means3D[3 * (size_t)i + 1], a.means3D[3 * (size_t)i + 2]);
        if (a.cov3D_precomp != nullptr) {
#pragma unroll
          for (int k = 0; k < 6; k++) c3[k] = a.cov3D_precomp[6 * (size_t)i + k];
        } else {
          quat_to_R(a.rotations[4 * (size_t)i], a.rotations[4 * (size_t)i + 1], a.rotations[4 * (size_t)i + 2],
                    a.rotations[4 * (size_t)i + 3], Rw);
#pragma unroll
          for (int k = 0; k < 3; k++) s[k] = a.scale_modifier * a.scales[3 * (size_t)i + k];
          cov3d_from_R(Rw, s, c3);
        }
      }
      view_backward<CAM == CAM_DEVFOV, DA>(a, cam, tanfov, m, c3, g, gm, gcov);
    }

    // ---- SH: dL/dsh written for every splat (zeros when invisible), direction term -> gm ----
    if (use_sh) {
      float gRGB[3] = {0.f, 0.f, 0.f};
      float B[16];
#pragma unroll
      for (int k = 0; k < 16; k++) B[k] = 0.f;
      if (visible) {
        const uint8_t cl = clamped[i];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) gRGB[ch] = ((cl >> ch) & 1) ? 0.f : gcol[ch];
        sh_dir_backward<BOUND>(a.sh_degree, cam.campos, m, my_sh, gRGB, B, gm);
      }
      // this thread is done reading its own row: overwrite it with the gradient row, then the block writes it out
      if (BOUND) {
        if (active && (!MC || visible)) {
          float* gdc_out = b.dL_dsh_dc + 3 * (size_t)i;
          put<MC>(gdc_out + 0, B[0] * gRGB[0]); put<MC>(gdc_out + 1, B[0] * gRGB[1]); put<MC>(gdc_out + 2, B[0] * gRGB[2]);
        }
        for (int k = 1; k < M; k++) {
          const float bk = (k < nb) ? B[k] : 0.f;
          my_sh[3 * (k - 1) + 0] = bk * gRGB[0];
          my_sh[3 * (k - 1) + 1] = bk * gRGB[1];
          my_sh[3 * (k - 1) + 2] = bk * gRGB[2];
        }
      } else {
        for (int k = 0; k < M; k++) {
          const float bk = (k < nb) ? B[k] : 0.f;
          my_sh[3 * k + 0] = bk * gRGB[0];
          my_sh[3 * k + 1] = bk * gRGB[1];
          my_sh[3 * k + 2] = bk * gRGB[2];
        }
      }
    }
  }
  if (stage_sh) {
    __syncthreads();
    float* dst = BOUND ? b.dL_dsh_rest : b.dL_dshs;
    if (dst != nullptr) stage_rows_out<PRE_NT, MC>(VIEWS ? shg_s : sh_s, dst, (size_t)row0, rows, sh_width, sh_stride);
    // multicast reductions are weak operations: order them before anything this grid's completion is used to
    // signal (the group barrier that follows the kernel on the stream)
    if (MC) __threadfence_system();
  }

  // ---- Sigma -> (scale, rotation) [-> binding chain] ----
  float g_xyz[3] = {gm[0], gm[1], gm[2]};
  float g_opacity_out = g_op;
  if (visible && from_sr)
    chain_backward<BOUND>(a, b, i, gcov, gm, g_op, Rw, s, act, ctx, face_scratch != nullptr, my_fg, gscale,
                          grot, g_xyz, g_opacity_out);

  if (BOUND && face_scratch != nullptr) {
    __syncthreads();
    stage_rows_out<PRE_NT>(fg_s, face_scratch, (size_t)row0, rows, GAB_FACE_GRAD_STRIDE, GAB_FACE_GRAD_STRIDE);
  }

  // ---- stores ----
  if (!active) return;
  const bool emit_param = !MC || visible;  // multicast mode: splats without gradient add nothing
  if (b.dL_dmeans3D != nullptr && emit_param) {
    put<MC>(b.dL_dmeans3D + 3 * (size_t)i + 0, g_xyz[0]);
    put<MC>(b.dL_dmeans3D + 3 * (size_t)i + 1, g_xyz[1]);
    put<MC>(b.dL_dmeans3D + 3 * (size_t)i + 2, g_xyz[2]);
  }
  if (b.dL_dopacity != nullptr && emit_param) put<MC>(b.dL_dopacity + i, g_opacity_out);
  if (b.dL_dscales != nullptr && emit_param) {
#pragma unroll
    for (int k = 0; k < 3; k++) put<MC>(b.dL_dscales + 3 * (size_t)i + k, gscale[k]);
  }
  if (b.dL_drotations != nullptr && emit_param) {
#pragma unroll
    for (int k = 0; k < 4; k++) put<MC>(b.dL_drotations + 4 * (size_t)i + k, grot[k]);
  }
  if constexpr (VIEWS) {
    if (b.dL_dsh_dc != nullptr) {
#pragma unroll
      for (int k = 0; k < 3; k++) b.dL_dsh_dc[3 * (size_t)i + k] = gdc[k];
    }
  } else {
    if (b.dL_dmeans2D != nullptr) {
      b.dL_dmeans2D[3 * (size_t)i + 0] = g2x;
      b.dL_dmeans2D[3 * (size_t)i + 1] = g2y;
      b.dL_dmeans2D[3 * (size_t)i + 2] = 0.f;
    }
    if (b.dL_dcolors != nullptr) {
#pragma unroll
      for (int k = 0; k < 3; k++) b.dL_dcolors[3 * (size_t)i + k] = gcol[k];
    }
    if (b.dL_dcov3D != nullptr) {
#pragma unroll
      for (int k = 0; k < 6; k++) b.dL_dcov3D[6 * (size_t)i + k] = gcov[k];
    }
  }
  if (MC) __threadfence_system();
}

// One 16-lane group per chunk (<= 64 splats of one face); lane c < 13 sums component c of the chunk's splats and
// adds it once to the face's output (several chunks only for faces with > 64 splats).
__global__ void __launch_bounds__(256) face_grad_reduce_kernel(int num_chunks, const int32_t* __restrict__ perm,
                                                               const int32_t* __restrict__ chunk_face,
                                                               const int32_t* __restrict__ chunk_start,
                                                               const int32_t* __restrict__ chunk_end,
                                                               const float* __restrict__ fg, float* __restrict__ d_fc,
                                                               float* __restrict__ d_fR, float* __restrict__ d_fs) {
  pdl_wait();
  pdl_trigger();
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 4, c = threadIdx.x & 15;
  if (g >= num_chunks || c >= GAB_FACE_GRAD_STRIDE) return;
  const int s0 = chunk_start[g], s1 = chunk_end[g];
  float acc = 0.f;
  int k = s0;
  for (; k + 4 <= s1; k += 4) {  // four independent gathers in flight
    const int i0 = perm[k], i1 = perm[k + 1], i2 = perm[k + 2], i3 = perm[k + 3];
    const float v0 = fg[(size_t)i0 * GAB_FACE_GRAD_STRIDE + c], v1 = fg[(size_t)i1 * GAB_FACE_GRAD_STRIDE + c];
    const float v2 = fg[(size_t)i2 * GAB_FACE_GRAD_STRIDE + c], v3 = fg[(size_t)i3 * GAB_FACE_GRAD_STRIDE + c];
    acc += (v0 + v1) + (v2 + v3);
  }
  for (; k < s1; k++) acc += fg[(size_t)perm[k] * GAB_FACE_GRAD_STRIDE + c];
  const size_t f = (size_t)chunk_face[g];
  float* dst = c < 3 ? (d_fc ? d_fc + 3 * f + c : nullptr)
                     : (c < 12 ? (d_fR ? d_fR + 9 * f + (c - 3) : nullptr) : (d_fs ? d_fs + f : nullptr));
  if (dst != nullptr) atomicAdd(dst, acc);
}

// one camera: multicast only with BOUND_RAW and without the depth plane (both refused by the caller)
template <int CAM>
static decltype(&preprocess_backward_kernel<true, false, CAM, false>) backward_instance(bool bound, bool mc, bool da) {
  if (da) return bound ? preprocess_backward_kernel<true, false, CAM, true> : preprocess_backward_kernel<false, false, CAM, true>;
  if (!bound) return preprocess_backward_kernel<false, false, CAM, false>;
  return mc ? preprocess_backward_kernel<true, true, CAM, false> : preprocess_backward_kernel<true, false, CAM, false>;
}

void launch_preprocess_backward(const gab200_backward_args& b, int views, const float* cameras, const float* tanfov,
                                const SplatAux* aux, const uint8_t* clamped, const float* g2d, float* face_scratch,
                                bool da, cudaStream_t stream) {
  const gab200_forward_args& a = *b.fwd;
  const int threads = PRE_NT, blocks = (a.P + threads - 1) / threads;
  if (blocks == 0) return;
  const bool bound = a.input_mode == GAB200_INPUT_BOUND_RAW;
  auto kernel = cameras != nullptr ? (da ? preprocess_backward_kernel<true, false, CAM_TABLE, true>
                                         : preprocess_backward_kernel<true, false, CAM_TABLE, false>)
                : tanfov != nullptr ? backward_instance<CAM_DEVFOV>(bound, b.grads_are_multicast, da)
                                    : backward_instance<CAM_ARGS>(bound, b.grads_are_multicast, da);
  launch_pdl(kernel, blocks, threads, 0, stream, b, a, views, cameras, tanfov, aux, clamped, g2d, face_scratch);
  if (face_scratch != nullptr && b.num_face_chunks > 0) {
    const int groups_per_block = 256 / 16;
    launch_pdl(face_grad_reduce_kernel, (b.num_face_chunks + groups_per_block - 1) / groups_per_block, 256, 0, stream,
               b.num_face_chunks, b.face_perm, b.face_chunk_face, b.face_chunk_start, b.face_chunk_end, face_scratch,
               b.dL_dface_center, b.dL_dface_orien_mat, b.dL_dface_scaling);
  }
}

}  // namespace gab
