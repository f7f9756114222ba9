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
  constexpr bool BOUND = true, DEVFOV = true, DEPTH = false;
#include "preprocess_bwd_views_splat.inc"
}

// gab200_backward_views_depth_alpha: preprocess_backward_views_kernel that also adds each view's dL/dz (g2d slot 9 of
// virtual splat k * P + i) to that view's dL/dmean through view k's own view-matrix row -- the camera row staged in
// shared memory for the view -- before the sums go on through Sigma -> (s, q), the binding chain and the face frame.
// Plain stores only.
__global__ void __launch_bounds__(PRE_NT) preprocess_backward_views_depth_kernel(gab200_backward_args b,
                                                                                gab200_forward_args a, int views,
                                                                                const float* __restrict__ cameras,
                                                                                const SplatAux* __restrict__ aux,
                                                                                const uint8_t* __restrict__ clamped,
                                                                                const float* __restrict__ g2d,
                                                                                float* __restrict__ face_scratch) {
  constexpr bool BOUND = true, DEVFOV = true, DEPTH = true;
#include "preprocess_bwd_views_splat.inc"
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
    launch_pdl(kernel, blocks, threads, 0, stream, b, a, rec, aux, clamped, g2d,
               a.input_mode == GAB200_INPUT_BOUND_RAW ? face_scratch : nullptr, tanfov);
  } else if (a.input_mode == GAB200_INPUT_BOUND_RAW) {
    auto kernel = b.grads_are_multicast
                      ? (dev ? preprocess_backward_kernel<true, true, true> : preprocess_backward_kernel<true, true, false>)
                      : (dev ? preprocess_backward_kernel<true, false, true> : preprocess_backward_kernel<true, false, false>);
    launch_pdl(kernel, blocks, threads, 0, stream, b, a, rec, aux, clamped, g2d, face_scratch, tanfov);
  } else {
    auto kernel = dev ? preprocess_backward_kernel<false, false, true> : preprocess_backward_kernel<false, false, false>;
    launch_pdl(kernel, blocks, threads, 0, stream, b, a, rec, aux, clamped, g2d, nullptr, tanfov);
  }
  if (face_scratch != nullptr && b.num_face_chunks > 0) {
    const int groups_per_block = 256 / 16;
    launch_pdl(face_grad_reduce_kernel, (b.num_face_chunks + groups_per_block - 1) / groups_per_block, 256, 0, stream,
               b.num_face_chunks, b.face_perm, b.face_chunk_face, b.face_chunk_start, b.face_chunk_end, face_scratch,
               b.dL_dface_center, b.dL_dface_orien_mat, b.dL_dface_scaling);
  }
}

void launch_preprocess_backward_views(const gab200_backward_args& b, int views, const float* cameras,
                                      const SplatAux* aux, const uint8_t* clamped, const float* g2d,
                                      float* face_scratch, cudaStream_t stream, bool depth) {
  const gab200_forward_args& a = *b.fwd;
  const int threads = PRE_NT, blocks = (a.P + threads - 1) / threads;
  if (blocks == 0) return;
  auto kernel = depth ? preprocess_backward_views_depth_kernel : preprocess_backward_views_kernel;
  launch_pdl(kernel, blocks, threads, 0, stream, b, a, views, cameras, aux, clamped, g2d, face_scratch);
  if (face_scratch != nullptr && b.num_face_chunks > 0) {
    const int groups_per_block = 256 / 16;
    launch_pdl(face_grad_reduce_kernel, (b.num_face_chunks + groups_per_block - 1) / groups_per_block, 256, 0, stream,
               b.num_face_chunks, b.face_perm, b.face_chunk_face, b.face_chunk_start, b.face_chunk_end, face_scratch,
               b.dL_dface_center, b.dL_dface_orien_mat, b.dL_dface_scaling);
  }
}

}  // namespace gab
