// face_frame.cu -- per-face frame of the posed mesh, forward and backward, as ONE kernel each.
// Replaces the ~25 eager launches of scene/flame_gaussian_model.py:137-147 + utils/graphics_utils.py:90-135
// (SURVEY.md 8a rows a1/a2, 8f rank 1):
//   a0 = norm(v1-v0); a1 = norm(a0 x (v2-v0)); a2 = -norm(a1 x a0); R = [a0 a1 a2] (columns)
//   scale = (|v1-v0| + |a2 . (v2-v0)|) / 2 ; centre = mean(v0,v1,v2);  norm(x) = x / sqrt(max(x.x, 1e-20))
// The quaternion detour of the reference (rotmat_to_unitquat) is not needed: the fused rasterizer composes matrices.
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

#define FF_EPS 1e-20f

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 ld3(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 operator*(float s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross3(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
// u = x / L, L = sqrt(max(x.x, eps)); returns L and whether the clamp was inactive
__device__ __forceinline__ V3 unit(V3 x, float& L, bool& free_) {
  const float d = dot3(x, x);
  free_ = d >= FF_EPS;
  L = sqrtf(fmaxf(d, FF_EPS));
  return (1.f / L) * x;
}
__device__ __forceinline__ V3 unit_bwd(V3 u, float L, bool free_, V3 g) {
  V3 r = (1.f / L) * g;
  if (free_) r = r - (dot3(u, g) / L) * u;
  return r;
}

__global__ void __launch_bounds__(256) face_frame_fwd_kernel(int F, const float* __restrict__ verts,
                                                             const int32_t* __restrict__ faces,
                                                             float* __restrict__ fc, float* __restrict__ fR,
                                                             float* __restrict__ fs) {
  pdl_wait();
  pdl_trigger();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const V3 v0 = ld3(verts + 3 * (size_t)faces[3 * f]), v1 = ld3(verts + 3 * (size_t)faces[3 * f + 1]),
           v2 = ld3(verts + 3 * (size_t)faces[3 * f + 2]);
  const V3 e01 = v1 - v0, e02 = v2 - v0;
  float L0, L1, L2;
  bool f0, f1, f2;
  const V3 a0 = unit(e01, L0, f0);
  const V3 a1 = unit(cross3(a0, e02), L1, f1);
  const V3 u2 = unit(cross3(a1, a0), L2, f2);
  const V3 a2 = -1.f * u2;
  float* R = fR + 9 * (size_t)f;
  R[0] = a0.x; R[1] = a1.x; R[2] = a2.x;
  R[3] = a0.y; R[4] = a1.y; R[5] = a2.y;
  R[6] = a0.z; R[7] = a1.z; R[8] = a2.z;
  fs[f] = (L0 + fabsf(dot3(a2, e02))) / 2.f;
  fc[3 * (size_t)f + 0] = (v0.x + v1.x + v2.x) / 3.f;
  fc[3 * (size_t)f + 1] = (v0.y + v1.y + v2.y) / 3.f;
  fc[3 * (size_t)f + 2] = (v0.z + v1.z + v2.z) / 3.f;
}

__global__ void __launch_bounds__(256) face_frame_bwd_kernel(int F, const float* __restrict__ verts,
                                                             const int32_t* __restrict__ faces,
                                                             const float* __restrict__ g_fc,
                                                             const float* __restrict__ g_fR,
                                                             const float* __restrict__ g_fs,
                                                             float* __restrict__ g_verts) {
  pdl_wait();
  pdl_trigger();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
  const V3 v0 = ld3(verts + 3 * (size_t)i0), v1 = ld3(verts + 3 * (size_t)i1), v2 = ld3(verts + 3 * (size_t)i2);
  const V3 e01 = v1 - v0, e02 = v2 - v0;
  float L0, L1, L2;
  bool f0, f1, f2;
  const V3 a0 = unit(e01, L0, f0);
  const V3 a1 = unit(cross3(a0, e02), L1, f1);
  const V3 u2 = unit(cross3(a1, a0), L2, f2);
  const V3 a2 = -1.f * u2;
  V3 ga0 = {0, 0, 0}, ga1 = {0, 0, 0}, ga2 = {0, 0, 0}, ge02 = {0, 0, 0};
  if (g_fR != nullptr) {
    const float* G = g_fR + 9 * (size_t)f;
    ga0 = {G[0], G[3], G[6]};
    ga1 = {G[1], G[4], G[7]};
    ga2 = {G[2], G[5], G[8]};
  }
  float gs = g_fs != nullptr ? g_fs[f] : 0.f;
  // scale = (L0 + |d|)/2, d = a2 . e02
  const float d = dot3(a2, e02);
  const float gd = 0.5f * gs * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
  ga2 = ga2 + gd * e02;
  ge02 = ge02 + gd * a2;
  // a2 = -unit(m), m = a1 x a0
  const V3 gm = unit_bwd(u2, L2, f2, -1.f * ga2);
  ga1 = ga1 + cross3(a0, gm);
  ga0 = ga0 + cross3(gm, a1);
  // a1 = unit(n), n = a0 x e02
  const V3 gn = unit_bwd(a1, L1, f1, ga1);
  ga0 = ga0 + cross3(e02, gn);
  ge02 = ge02 + cross3(gn, a0);
  // a0 = unit(e01); L0 also feeds the scale
  V3 ge01 = unit_bwd(a0, L0, f0, ga0);
  if (f0) ge01 = ge01 + (0.5f * gs) * a0;
  V3 gc = {0, 0, 0};
  if (g_fc != nullptr) gc = (1.f / 3.f) * ld3(g_fc + 3 * (size_t)f);
  const V3 gv1 = ge01 + gc, gv2 = ge02 + gc, gv0 = gc - (ge01 + ge02);
  atomicAdd(g_verts + 3 * (size_t)i0 + 0, gv0.x); atomicAdd(g_verts + 3 * (size_t)i0 + 1, gv0.y); atomicAdd(g_verts + 3 * (size_t)i0 + 2, gv0.z);
  atomicAdd(g_verts + 3 * (size_t)i1 + 0, gv1.x); atomicAdd(g_verts + 3 * (size_t)i1 + 1, gv1.y); atomicAdd(g_verts + 3 * (size_t)i1 + 2, gv1.z);
  atomicAdd(g_verts + 3 * (size_t)i2 + 0, gv2.x); atomicAdd(g_verts + 3 * (size_t)i2 + 1, gv2.y); atomicAdd(g_verts + 3 * (size_t)i2 + 2, gv2.z);
}

void launch_face_frame_forward(int F, const float* verts, const int32_t* faces, float* fc, float* fR, float* fs,
                               cudaStream_t stream) {
  if (F == 0) return;
  launch_pdl(face_frame_fwd_kernel, (F + 255) / 256, 256, 0, stream, F, verts, faces, fc, fR, fs);
}
void launch_face_frame_backward(int F, const float* verts, const int32_t* faces, const float* g_fc, const float* g_fR,
                                const float* g_fs, float* g_verts, cudaStream_t stream) {
  if (F == 0) return;
  launch_pdl(face_frame_bwd_kernel, (F + 255) / 256, 256, 0, stream, F, verts, faces, g_fc, g_fR, g_fs, g_verts);
}

}  // namespace gab
