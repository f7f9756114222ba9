// densify.cu -- densify_and_prune of the splat arrays with the Adam-state surgery fused (SURVEY.md 8f rank 3).
//
// Replaces, per densification step, the reference's Python sequence (scene/gaussian_model.py:426-519 with the
// optimizer surgery of :334-419): clone the small high-gradient splats, split the large ones into two sampled
// children, prune the parents, prune by opacity / world size -- each a boolean-mask indexing + torch.cat over six
// parameter tensors and their exp_avg / exp_avg_sq, with binding / binding_counter bookkeeping in between
// (~150 eager launches and three full copies of 3 x 59 floats per splat).
//
// Every output row is a kept original, a clone, or a split child of ONE input row, so the whole sequence is a gather:
//   classify_kernel  per splat: clone / split / prune-candidate flags (+ the children's) and, per face, the change of
//                    its splat count and the number of prune candidates            [2 atomics per affected splat]
//   decide_kernel    the "every face keeps a splat" rule (all-or-nothing per face, :375-380) -> three 0/1 counts per
//                    splat (kept original, kept clone, kept child pair) + split-parent marker
//   cub::DeviceScan  four exclusive sums -> output positions; the totals go to the host (ONE sync: the caller has
//                    to size the outputs)
//   source_kernel    output row -> (input row, kind); kept children also get their noise rows
//   gather_kernel    ALL 18 arrays (6 parameters + 12 Adam moments) in one launch, coalesced over output elements:
//                    originals copy parameter and moments, clones / children copy the parameter and get zero moments
//   children_kernel  position = R(normalize(q)) (noise * world scale) + position, scale = log(((exp(s) fs) / fs) / 1.6)
//   recount_kernel   binding_counter of the result
// Compulsory traffic: read P x (236 + 472) B (parameters + moments of the kept originals), write P' x 708 B.
#include <cub/cub.cuh>

#include "common.cuh"
#include "kernels.cuh"

namespace gab {

enum : uint32_t { DF_CLONE = 1, DF_SPLIT = 2, DF_CRIT = 4, DF_CRIT_CHILD = 8 };

// torch.max(dim=1) of a scale triple: a NaN component makes the maximum NaN (fmaxf would drop it), and a NaN maximum
// compares false, so such a splat is never cloned, split or pruned for its size.
__device__ __forceinline__ float max3_nan(const float v[3]) {
  float m = v[0];
#pragma unroll
  for (int k = 1; k < 3; k++) m = (v[k] > m || isnan(v[k])) ? v[k] : m;
  return m;
}

__device__ __forceinline__ float world_scale_max(const gab200_densify_args& a, int i, float fs, float e[3]) {
#pragma unroll
  for (int k = 0; k < 3; k++) e[k] = expf(a.scaling[3 * (size_t)i + k]) * fs;  // get_scaling (scene/gaussian_model.py:113-123)
  return max3_nan(e);
}

// thr = f32(percent_dense * extent), big = f32(0.1 * extent), formed in double on the host: see launch_densify_plan.
__global__ void __launch_bounds__(256) densify_classify_kernel(gab200_densify_args a, float thr, float big,
                                                               uint32_t* __restrict__ flags,
                                                               int32_t* __restrict__ face_delta,
                                                               int32_t* __restrict__ face_cand) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  float g = a.xyz_gradient_accum[i] / a.denom[i];
  if (isnan(g)) g = 0.f;  // grads[grads.isnan()] = 0.0
  const bool bound = a.binding != nullptr;
  const int f = bound ? a.binding[i] : 0;
  const float fs = bound ? a.face_scaling[f] : 1.f;
  float e[3];
  const float smax = world_scale_max(a, i, fs, e);
  const bool clone = fabsf(g) >= a.grad_threshold && smax <= thr;
  const bool split = g >= a.grad_threshold && smax > thr;
  const float op = 1.0f / (1.0f + expf(-a.opacity[i]));
  const bool ws = a.max_screen_size > 0.f;  // the radius criterion itself can never fire: see oracle/densify.py
  const bool crit = op < a.min_opacity || (ws && smax > big);
  float child[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float base = bound ? e[k] / fs : e[k];
    const float ns = logf(base / 1.6f);  // scaling_inverse_activation(... / (0.8 * N)), N = 2
    child[k] = expf(ns) * fs;
  }
  const bool crit_child = op < a.min_opacity || (ws && max3_nan(child) > big);
  flags[i] = (clone ? DF_CLONE : 0u) | (split ? DF_SPLIT : 0u) | (crit ? DF_CRIT : 0u) | (crit_child ? DF_CRIT_CHILD : 0u);
  if (bound) {
    if (clone || split) atomicAdd(face_delta + f, 1);  // + clone, or + 2 children - 1 parent
    const int cand = ((!split && crit) ? 1 : 0) + ((clone && crit) ? 1 : 0) + ((split && crit_child) ? 2 : 0);
    if (cand) atomicAdd(face_cand + f, cand);
  }
}

__global__ void __launch_bounds__(256) densify_decide_kernel(gab200_densify_args a, const uint32_t* __restrict__ flags,
                                                             const int32_t* __restrict__ face_delta,
                                                             const int32_t* __restrict__ face_cand,
                                                             uint32_t* __restrict__ cnt /* [4][P] */) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  const uint32_t fl = flags[i];
  bool ok = true;
  if (a.binding != nullptr) {
    const int f = a.binding[i];
    ok = (a.binding_counter[f] + face_delta[f] - face_cand[f]) > 0;
  }
  const bool clone = fl & DF_CLONE, split = fl & DF_SPLIT;
  const bool pr = (fl & DF_CRIT) && ok, prc = (fl & DF_CRIT_CHILD) && ok;
  cnt[i] = (!split && !pr) ? 1u : 0u;
  cnt[(size_t)a.P + i] = (clone && !pr) ? 1u : 0u;
  cnt[2 * (size_t)a.P + i] = (split && !prc) ? 1u : 0u;
  cnt[3 * (size_t)a.P + i] = split ? 1u : 0u;
}

// totals[0..3] = kept originals, kept clones, kept child PAIRS, split parents
__global__ void densify_totals_kernel(int P, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ pos,
                                      uint32_t* __restrict__ totals) {
  const int k = threadIdx.x;
  if (k < 4) totals[k] = P > 0 ? pos[(size_t)k * P + P - 1] + cnt[(size_t)k * P + P - 1] : 0u;
}

// src[row'] = input row; kind[row'] = 0 original, 1 clone, 2 / 3 first / second child; noise_row[child pair slot]
__global__ void __launch_bounds__(256) densify_source_kernel(int P, const uint32_t* __restrict__ cnt,
                                                             const uint32_t* __restrict__ pos,
                                                             const uint32_t* __restrict__ totals,
                                                             int32_t* __restrict__ src, uint8_t* __restrict__ kind,
                                                             int32_t* __restrict__ noise_row) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const uint32_t n_o = totals[0], n_c = totals[1], n_ch = totals[2];
  if (cnt[i]) {
    src[pos[i]] = i;
    kind[pos[i]] = 0;
  }
  if (cnt[(size_t)P + i]) {
    const uint32_t o = n_o + pos[(size_t)P + i];
    src[o] = i;
    kind[o] = 1;
  }
  if (cnt[2 * (size_t)P + i]) {
    const uint32_t slot = pos[2 * (size_t)P + i];
    const uint32_t o = n_o + n_c + slot;
    src[o] = i;
    kind[o] = 2;
    src[o + n_ch] = i;
    kind[o + n_ch] = 3;
    noise_row[slot] = (int32_t)pos[3 * (size_t)P + i];  // rank among ALL split parents: the reference's sample index
  }
}

struct GatherBatch {
  const float* in[18];
  float* out[18];
  int width[18];
  int zero_new[18];  // moments: rows that are not kept originals are zero
};
__global__ void __launch_bounds__(256) densify_gather_kernel(GatherBatch b, int P_out, const int32_t* __restrict__ src,
                                                             const uint8_t* __restrict__ kind) {
  const int arr = blockIdx.y;
  const int w = b.width[arr];
  if (b.in[arr] == nullptr || b.out[arr] == nullptr || w == 0) return;
  const size_t total = (size_t)P_out * w;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / w;
    const int col = (int)(e - row * w);
    const bool zero = b.zero_new[arr] && kind[row] != 0;
    b.out[arr][e] = zero ? 0.f : b.in[arr][(size_t)src[row] * w + col];
  }
}

__global__ void __launch_bounds__(256) densify_children_kernel(gab200_densify_args a, const uint32_t* __restrict__ totals,
                                                               const int32_t* __restrict__ src,
                                                               const int32_t* __restrict__ noise_row,
                                                               const float* __restrict__ noise, float* __restrict__ xyz_out,
                                                               float* __restrict__ scaling_out) {
  const uint32_t n_o = totals[0], n_c = totals[1], n_ch = totals[2], S = totals[3];
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * n_ch) return;
  const uint32_t copy = t >= n_ch ? 1u : 0u, slot = t - copy * n_ch;
  const size_t o = (size_t)n_o + n_c + t;
  const int i = src[o];
  const bool bound = a.binding != nullptr;
  const float fs = bound ? a.face_scaling[a.binding[i]] : 1.f;
  float e[3];
  world_scale_max(a, i, fs, e);
  const float* nz = noise + 3 * ((size_t)noise_row[slot] + (size_t)copy * S);
  const float s0 = nz[0] * e[0], s1 = nz[1] * e[1], s2 = nz[2] * e[2];  // torch.normal(mean = 0, std = get_scaling)
  // build_rotation (utils/general_utils.py:78-99): plain normalisation, no epsilon
  const float qr = a.rotation[4 * (size_t)i], qx = a.rotation[4 * (size_t)i + 1], qy = a.rotation[4 * (size_t)i + 2],
              qz = a.rotation[4 * (size_t)i + 3];
  const float n = sqrtf(qr * qr + qx * qx + qy * qy + qz * qz);
  const float r = qr / n, x = qx / n, y = qy / n, z = qz / n;
  const float R00 = 1.f - 2.f * (y * y + z * z), R01 = 2.f * (x * y - r * z), R02 = 2.f * (x * z + r * y);
  const float R10 = 2.f * (x * y + r * z), R11 = 1.f - 2.f * (x * x + z * z), R12 = 2.f * (y * z - r * x);
  const float R20 = 2.f * (x * z - r * y), R21 = 2.f * (y * z + r * x), R22 = 1.f - 2.f * (x * x + y * y);
  xyz_out[3 * o + 0] = (R00 * s0 + R01 * s1 + R02 * s2) + a.xyz[3 * (size_t)i + 0];
  xyz_out[3 * o + 1] = (R10 * s0 + R11 * s1 + R12 * s2) + a.xyz[3 * (size_t)i + 1];
  xyz_out[3 * o + 2] = (R20 * s0 + R21 * s1 + R22 * s2) + a.xyz[3 * (size_t)i + 2];
#pragma unroll
  for (int k = 0; k < 3; k++) scaling_out[3 * o + k] = logf((bound ? e[k] / fs : e[k]) / 1.6f);
}

__global__ void __launch_bounds__(256) densify_binding_kernel(int P_out, const int32_t* __restrict__ src,
                                                              const int32_t* __restrict__ binding_in,
                                                              int32_t* __restrict__ binding_out,
                                                              int32_t* __restrict__ counter_out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= P_out) return;
  const int f = binding_in[src[o]];
  binding_out[o] = f;
  atomicAdd(counter_out + f, 1);
}

size_t densify_scratch_bytes(int P, int F) {
  Carver c(nullptr);
  c.take<uint32_t>((size_t)P);          // flags
  c.take<uint32_t>(4 * (size_t)P);      // counts
  c.take<uint32_t>(4 * (size_t)P);      // positions
  c.take<int32_t>(2 * (size_t)F);       // face delta | candidates
  c.take<uint32_t>(8);                  // totals
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const uint32_t*)nullptr, (uint32_t*)nullptr, P > 0 ? P : 1);
  c.take<char>(temp);
  return c.bytes();
}

struct DensifyScratch {
  uint32_t *flags, *cnt, *pos, *totals;
  int32_t* face;
  void* scan_temp;
  size_t scan_bytes;
};
static DensifyScratch carve_densify(void* base, int P, int F) {
  DensifyScratch s;
  Carver c(base);
  s.flags = c.take<uint32_t>((size_t)P);
  s.cnt = c.take<uint32_t>(4 * (size_t)P);
  s.pos = c.take<uint32_t>(4 * (size_t)P);
  s.face = c.take<int32_t>(2 * (size_t)F);
  s.totals = c.take<uint32_t>(8);
  s.scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, s.scan_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, P > 0 ? P : 1);
  s.scan_temp = c.take<char>(s.scan_bytes);
  return s;
}

cudaError_t launch_densify_plan(const gab200_densify_args& a, double extent, double percent_dense, cudaStream_t stream) {
  const int P = a.P, F = a.binding != nullptr ? a.num_faces : 0;
  DensifyScratch s = carve_densify(a.scratch, P, F);
  cudaError_t e;
  if (F > 0 && (e = cudaMemsetAsync(s.face, 0, sizeof(int32_t) * 2 * (size_t)F, stream)) != cudaSuccess) return e;
  if (P == 0) {
    if ((e = cudaMemsetAsync(s.totals, 0, sizeof(uint32_t) * 8, stream)) != cudaSuccess) return e;
  } else {
    // The reference compares float32 scales with Python products, formed in double and rounded once; a float product
    // of the rounded factors differs from that by an ulp for about a third of all extents.
    const float thr = (float)(percent_dense * extent), big = (float)(0.1 * extent);
    const int blocks = (P + 255) / 256;
    densify_classify_kernel<<<blocks, 256, 0, stream>>>(a, thr, big, s.flags, s.face, s.face + F);
    count_launch();
    densify_decide_kernel<<<blocks, 256, 0, stream>>>(a, s.flags, s.face, s.face + F, s.cnt);
    count_launch();
    for (int k = 0; k < 4; k++) {
      size_t bytes = s.scan_bytes;
      e = cub::DeviceScan::ExclusiveSum(s.scan_temp, bytes, s.cnt + (size_t)k * P, s.pos + (size_t)k * P, P, stream);
      if (e != cudaSuccess) return e;
      count_launch();
    }
    densify_totals_kernel<<<1, 32, 0, stream>>>(P, s.cnt, s.pos, s.totals);
    count_launch();
  }
  return cudaMemcpyAsync(a.totals_host, s.totals, sizeof(uint32_t) * 4, cudaMemcpyDeviceToHost, stream);
}

cudaError_t launch_densify_apply(const gab200_densify_args& a, const gab200_densify_out& o, cudaStream_t stream) {
  const int P = a.P, F = a.binding != nullptr ? a.num_faces : 0;
  DensifyScratch s = carve_densify(a.scratch, P, F);
  const int P_out = o.P_out;
  // also when P_out = 0: the counters of a bound model without splats are all zero (its binding pointer may be NULL)
  const int F_counter = (F > 0 || (P == 0 && a.num_faces > 0)) ? a.num_faces : 0;
  if (F_counter > 0 && o.binding_counter != nullptr) {
    cudaError_t e = cudaMemsetAsync(o.binding_counter, 0, sizeof(int32_t) * (size_t)F_counter, stream);
    if (e != cudaSuccess) return e;
  }
  if (P_out == 0 || P == 0) return cudaSuccess;
  const int blocks = (P + 255) / 256;
  densify_source_kernel<<<blocks, 256, 0, stream>>>(P, s.cnt, s.pos, s.totals, o.src_scratch, o.kind_scratch,
                                                    o.noise_row_scratch);
  count_launch();
  GatherBatch b;
  const float* in_p[6] = {a.xyz, a.rotation, a.scaling, a.opacity, a.f_dc, a.f_rest};
  float* out_p[6] = {o.xyz, o.rotation, o.scaling, o.opacity, o.f_dc, o.f_rest};
  const int w[6] = {3, 4, 3, 1, 3, a.sh_rest_width};
  for (int k = 0; k < 6; k++) {
    b.in[k] = in_p[k]; b.out[k] = out_p[k]; b.width[k] = w[k]; b.zero_new[k] = 0;
    b.in[6 + k] = a.exp_avg[k]; b.out[6 + k] = o.exp_avg[k]; b.width[6 + k] = w[k]; b.zero_new[6 + k] = 1;
    b.in[12 + k] = a.exp_avg_sq[k]; b.out[12 + k] = o.exp_avg_sq[k]; b.width[12 + k] = w[k]; b.zero_new[12 + k] = 1;
  }
  int64_t gblocks = ((int64_t)P_out * (a.sh_rest_width > 4 ? a.sh_rest_width : 4) / 4 + 255) / 256;
  if (gblocks < 1) gblocks = 1;
  if (gblocks > GAB_NUM_SMS * 16) gblocks = GAB_NUM_SMS * 16;
  densify_gather_kernel<<<dim3((unsigned)gblocks, 18), 256, 0, stream>>>(b, P_out, o.src_scratch, o.kind_scratch);
  count_launch();
  if (o.n_child_rows > 0) {
    densify_children_kernel<<<(o.n_child_rows + 255) / 256, 256, 0, stream>>>(a, s.totals, o.src_scratch,
                                                                             o.noise_row_scratch, o.noise, o.xyz, o.scaling);
    count_launch();
  }
  if (F > 0) {
    densify_binding_kernel<<<(P_out + 255) / 256, 256, 0, stream>>>(P_out, o.src_scratch, a.binding, o.binding,
                                                                     o.binding_counter);
    count_launch();
  }
  return cudaSuccess;
}

// The statistics densify_and_prune consumes, accumulated once per rendered frame (train.py:197,
// scene/gaussian_model.py:517-519) without the reference's two boolean-mask index passes (each a nonzero(): a host
// wait).  Per splat: read the x, y of the view-space gradient (8 B), radii (4 B) and the three statistics (12 B);
// write the statistics (12 B) where radii > 0.
__global__ void __launch_bounds__(256) densify_stats_kernel(int P, const float* __restrict__ vgrad,
                                                            const int32_t* __restrict__ radii, float* __restrict__ accum,
                                                            float* __restrict__ denom, float* __restrict__ max_radii,
                                                            const int32_t* __restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int r = radii[i];
  if (r <= 0) return;
  max_radii[i] = fmaxf(max_radii[i], (float)r);
  const float gx = vgrad[3 * (size_t)i], gy = vgrad[3 * (size_t)i + 1];
  accum[i] += sqrtf(fmaf(gy, gy, gx * gx));  // torch.norm(grad[:, :2], dim=-1)
  denom[i] += 1.f;
}

void launch_densify_stats(int P, const float* vgrad, const int32_t* radii, float* accum, float* denom, float* max_radii,
                          const int32_t* skip, cudaStream_t stream) {
  if (P <= 0) return;
  densify_stats_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, vgrad, radii, accum, denom, max_radii, skip);
  count_launch();
}

}  // namespace gab
