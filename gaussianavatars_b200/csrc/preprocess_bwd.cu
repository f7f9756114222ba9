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

// DEVFOV: (tanfovx, tanfovy) from the device float[2] `tanfov` the forward read (gab200_backward_device_fov).
template <bool BOUND, bool MC, bool DEVFOV>
__global__ void __launch_bounds__(PRE_NT, 12) preprocess_backward_kernel(gab200_backward_args b, gab200_forward_args a,
                                                                  const SplatRec* __restrict__ rec,
                                                                  const SplatAux* __restrict__ aux,
                                                                  const uint8_t* __restrict__ clamped,
                                                                  const float* __restrict__ g2d,
                                                                  float* __restrict__ face_scratch,
                                                                  const float* __restrict__ tanfov) {
  constexpr bool DEPTH = false;
#include "preprocess_bwd_splat.inc"
}

// gab200_backward_depth_alpha: preprocess_backward_kernel that also adds dL/dz (g2d slot 9) to dL/dmean through the third
// row of the view matrix, before the binding chain.  Plain stores only.  Bounded for 8 CTAs per SM (up to 128 registers):
// under the 12 of preprocess_backward_kernel (80 registers) its BOUND instances spill.
template <bool BOUND, bool DEVFOV>
__global__ void __launch_bounds__(PRE_NT, 8) preprocess_backward_depth_kernel(gab200_backward_args b,
                                                                        gab200_forward_args a,
                                                                        const SplatRec* __restrict__ rec,
                                                                        const SplatAux* __restrict__ aux,
                                                                        const uint8_t* __restrict__ clamped,
                                                                        const float* __restrict__ g2d,
                                                                        float* __restrict__ face_scratch,
                                                                        const float* __restrict__ tanfov) {
  constexpr bool MC = false, DEPTH = true;
#include "preprocess_bwd_splat.inc"
}

// gab200_backward_views (BOUND_RAW): one thread per REAL splat i walks the views in order.  Per view k it stages camera
// row k, reads the 2-D gradients, radius and clamp bits of virtual splat k * P + i, writes dL/dmeans2D row (k, i) and
// adds that view's dL/dSigma, dL/dmean (direction term of the SH colour included), dL/dopacity and SH gradients to
// sums kept in registers (SH: a second shared-memory tile beside the staged coefficients).  Every step after those is
// linear in them, so the binding chain and the face-frame gradients run once, on the sums, and every gradient is
// stored once: no cross-view atomics and no per-view gradient scratch.  The binding, the parameter loads and the staged
// SH rows serve all views.  A view in which the splat is not visible (radius 0 -- also every splat of a view whose
// tan(FoV/2) is invalid) adds nothing.
__global__ void __launch_bounds__(PRE_NT) preprocess_backward_views_kernel(gab200_backward_args b, gab200_forward_args a,
                                                                          int views, const float* __restrict__ cameras,
                                                                          const SplatAux* __restrict__ aux,
                                                                          const uint8_t* __restrict__ clamped,
                                                                          const float* __restrict__ g2d,
                                                                          float* __restrict__ face_scratch) {
  constexpr bool BOUND = true, DEVFOV = true;
  __shared__ Camera cam;
  __shared__ float fg_s[PRE_NT * GAB_FACE_GRAD_STRIDE];
  __shared__ float sh_s[PRE_NT * SH_SMEM_STRIDE_MAX];   // SH coefficients (read by every view's direction term)
  __shared__ float shg_s[PRE_NT * SH_SMEM_STRIDE_MAX];  // SH gradients summed over the views
  float* my_fg = fg_s + threadIdx.x * GAB_FACE_GRAD_STRIDE;
  if (face_scratch != nullptr) {
#pragma unroll
    for (int k = 0; k < GAB_FACE_GRAD_STRIDE; k++) my_fg[k] = 0.f;
  }
  const int M = a.sh_coeffs;
  const int sh_width = 3 * (M - 1);
  const int sh_stride = sh_width | 1;
  const int row0 = blockIdx.x * PRE_NT;
  const int rows = min(PRE_NT, a.P - row0);
  const bool stage_sh = a.sh_rest != nullptr && sh_width > 0;
  float* my_sh = sh_s + threadIdx.x * sh_stride;
  float* my_shg = shg_s + threadIdx.x * sh_stride;
  for (int k = 0; k < sh_width; k++) my_shg[k] = 0.f;
  if (stage_sh && a.sh_degree > 0) stage_rows_in<PRE_NT>(sh_s, a.sh_rest, (size_t)row0, rows, sh_width, sh_stride);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = idx < a.P;
  const int i = active ? idx : a.P - 1;
  const int W = a.image_width, H = a.image_height;
  const int nb = (a.sh_degree + 1) * (a.sh_degree + 1);

  Activated act;
  BindCtx ctx;
  bind_activate(a, i, act, ctx);
  const float3 m = act.mean;
  float Rw[9], s[3], c3[6];
#pragma unroll
  for (int k = 0; k < 9; k++) Rw[k] = act.R[k];
#pragma unroll
  for (int k = 0; k < 3; k++) s[k] = a.scale_modifier * act.s[k];
  cov3d_from_R(Rw, s, c3);

  float sgm[3] = {0.f, 0.f, 0.f}, sgcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float g_op = 0.f, gdc[3] = {0.f, 0.f, 0.f};
  bool any_visible = false;
  for (int view = 0; view < views; view++) {
    const float* row = cameras + (size_t)view * GAB200_CAMERA_FLOATS;
    __syncthreads();  // the previous view's camera is no longer read (first view: the SH rows are staged)
    {
      const int t = threadIdx.x;
      if (t < 16) cam.V[t] = row[t];
      else if (t < 32) cam.Pm[t - 16] = row[t];
      else if (t < 35) cam.campos[t - 32] = row[t];
    }
    __syncthreads();
    const size_t vi = (size_t)view * a.P + i;
    const bool visible = active && aux[vi].radius > 0;
    float g2x = 0.f, g2y = 0.f;
    if (visible) {
      any_visible = true;
      const float* g = g2d + vi * GAB_G2D_STRIDE;
      g2x = g[0]; g2y = g[1];
      const float gA = g[2], gB = g[3], gC = g[4];
      g_op += g[5];
      const float gcol[3] = {g[6], g[7], g[8]};
      const float* tanfov = row + 35;
      float gm[3] = {0.f, 0.f, 0.f}, gcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#include "preprocess_bwd_view.inc"
      if (a.colors_precomp == nullptr) {
        float gRGB[3];
        float B[16];
#pragma unroll
        for (int k = 0; k < 16; k++) B[k] = 0.f;
        const uint8_t cl = clamped[vi];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) gRGB[ch] = ((cl >> ch) & 1) ? 0.f : gcol[ch];
#include "preprocess_bwd_shdir.inc"
#pragma unroll
        for (int ch = 0; ch < 3; ch++) gdc[ch] += B[0] * gRGB[ch];
        for (int k = 1; k < nb && k < M; k++) {
          my_shg[3 * (k - 1) + 0] += B[k] * gRGB[0];
          my_shg[3 * (k - 1) + 1] += B[k] * gRGB[1];
          my_shg[3 * (k - 1) + 2] += B[k] * gRGB[2];
        }
      }
#pragma unroll
      for (int k = 0; k < 3; k++) sgm[k] += gm[k];
#pragma unroll
      for (int k = 0; k < 6; k++) sgcov[k] += gcov[k];
    }
    if (active && b.dL_dmeans2D != nullptr) {
      b.dL_dmeans2D[3 * vi + 0] = g2x;
      b.dL_dmeans2D[3 * vi + 1] = g2y;
      b.dL_dmeans2D[3 * vi + 2] = 0.f;
    }
  }

  float gscale[3] = {0.f, 0.f, 0.f}, grot[4] = {0.f, 0.f, 0.f, 0.f};
  float g_xyz[3] = {0.f, 0.f, 0.f};
  float g_opacity_out = 0.f;
  if (any_visible) {
    const float(&gm)[3] = sgm;
    const float(&gcov)[6] = sgcov;
#include "preprocess_bwd_chain.inc"
  }
  if (stage_sh) {
    __syncthreads();
    if (b.dL_dsh_rest != nullptr) stage_rows_out<PRE_NT>(shg_s, b.dL_dsh_rest, (size_t)row0, rows, sh_width, sh_stride);
  }
  if (face_scratch != nullptr) {
    __syncthreads();
    stage_rows_out<PRE_NT>(fg_s, face_scratch, (size_t)row0, rows, GAB_FACE_GRAD_STRIDE, GAB_FACE_GRAD_STRIDE);
  }

  if (!active) return;
  if (b.dL_dmeans3D != nullptr) {
#pragma unroll
    for (int k = 0; k < 3; k++) b.dL_dmeans3D[3 * (size_t)i + k] = g_xyz[k];
  }
  if (b.dL_dopacity != nullptr) b.dL_dopacity[i] = g_opacity_out;
  if (b.dL_dsh_dc != nullptr) {
#pragma unroll
    for (int k = 0; k < 3; k++) b.dL_dsh_dc[3 * (size_t)i + k] = gdc[k];
  }
  if (b.dL_dscales != nullptr) {
#pragma unroll
    for (int k = 0; k < 3; k++) b.dL_dscales[3 * (size_t)i + k] = gscale[k];
  }
  if (b.dL_drotations != nullptr) {
#pragma unroll
    for (int k = 0; k < 4; k++) b.dL_drotations[4 * (size_t)i + k] = grot[k];
  }
}

// One 16-lane group per chunk (<= 64 splats of one face); lane c < 13 sums component c of the chunk's splats and
// adds it once to the face's output (several chunks only for faces with > 64 splats).
__global__ void __launch_bounds__(256) face_grad_reduce_kernel(int num_chunks, const int32_t* __restrict__ perm,
                                                               const int32_t* __restrict__ chunk_face,
                                                               const int32_t* __restrict__ chunk_start,
                                                               const int32_t* __restrict__ chunk_end,
                                                               const float* __restrict__ fg, float* __restrict__ d_fc,
                                                               float* __restrict__ d_fR, float* __restrict__ d_fs) {
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

void launch_preprocess_backward(const gab200_backward_args& b, const SplatRec* rec, const SplatAux* aux,
                                const uint8_t* clamped, const float* g2d, float* face_scratch, const float* tanfov,
                                cudaStream_t stream, bool depth) {
  const gab200_forward_args& a = *b.fwd;
  const int threads = PRE_NT, blocks = (a.P + threads - 1) / threads;
  if (blocks == 0) return;
  const bool dev = tanfov != nullptr;
  if (depth) {  // multicast refused by the caller
    auto kernel = a.input_mode == GAB200_INPUT_BOUND_RAW
                      ? (dev ? preprocess_backward_depth_kernel<true, true> : preprocess_backward_depth_kernel<true, false>)
                      : (dev ? preprocess_backward_depth_kernel<false, true> : preprocess_backward_depth_kernel<false, false>);
    kernel<<<blocks, threads, 0, stream>>>(b, a, rec, aux, clamped, g2d,
                                           a.input_mode == GAB200_INPUT_BOUND_RAW ? face_scratch : nullptr, tanfov);
  } else if (a.input_mode == GAB200_INPUT_BOUND_RAW) {
    auto kernel = b.grads_are_multicast
                      ? (dev ? preprocess_backward_kernel<true, true, true> : preprocess_backward_kernel<true, true, false>)
                      : (dev ? preprocess_backward_kernel<true, false, true> : preprocess_backward_kernel<true, false, false>);
    kernel<<<blocks, threads, 0, stream>>>(b, a, rec, aux, clamped, g2d, face_scratch, tanfov);
  } else {
    auto kernel = dev ? preprocess_backward_kernel<false, false, true> : preprocess_backward_kernel<false, false, false>;
    kernel<<<blocks, threads, 0, stream>>>(b, a, rec, aux, clamped, g2d, nullptr, tanfov);
  }
  count_launch();
  if (face_scratch != nullptr && b.num_face_chunks > 0) {
    const int groups_per_block = 256 / 16;
    face_grad_reduce_kernel<<<(b.num_face_chunks + groups_per_block - 1) / groups_per_block, 256, 0, stream>>>(
        b.num_face_chunks, b.face_perm, b.face_chunk_face, b.face_chunk_start, b.face_chunk_end, face_scratch,
        b.dL_dface_center, b.dL_dface_orien_mat, b.dL_dface_scaling);
    count_launch();
  }
}

void launch_preprocess_backward_views(const gab200_backward_args& b, int views, const float* cameras,
                                      const SplatAux* aux, const uint8_t* clamped, const float* g2d,
                                      float* face_scratch, cudaStream_t stream) {
  const gab200_forward_args& a = *b.fwd;
  const int threads = PRE_NT, blocks = (a.P + threads - 1) / threads;
  if (blocks == 0) return;
  preprocess_backward_views_kernel<<<blocks, threads, 0, stream>>>(b, a, views, cameras, aux, clamped, g2d,
                                                                   face_scratch);
  count_launch();
  if (face_scratch != nullptr && b.num_face_chunks > 0) {
    const int groups_per_block = 256 / 16;
    face_grad_reduce_kernel<<<(b.num_face_chunks + groups_per_block - 1) / groups_per_block, 256, 0, stream>>>(
        b.num_face_chunks, b.face_perm, b.face_chunk_face, b.face_chunk_start, b.face_chunk_end, face_scratch,
        b.dL_dface_center, b.dL_dface_orien_mat, b.dL_dface_scaling);
    count_launch();
  }
}

}  // namespace gab
