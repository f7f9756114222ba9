// Shared device-side definitions for the gab200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gab200_rasterizer.h"

#define GAB_TILE 16                 // tile edge in pixels (binning granularity of the reference: 16x16)
#define GAB_TILE_PIX (GAB_TILE * GAB_TILE)
// SMs of the H100 SXM: sizes the persistent and capped grids (all grid-stride loops, so correct on any SM count)
#define GAB_NUM_SMS 132

namespace gab {

// Per-splat screen-space record written by preprocess and gathered by both blend kernels.
// 48 B = three 16-B quads so that one splat is three LDG.128 / cp.async.16:
//   q0 = (px, py, A', B')   q1 = (C', opacity, r, g)   q2 = (b, rx, ry, 0)
// with the conic pre-scaled for the blend exponent in log2 units: (A',B',C') = (-conic.xx/2, -conic.xy, -conic.yy/2)*log2 e
// (rx, ry) = half extents of the axis-aligned box around the region where the splat can reach alpha >= 1/255
// (negative: nowhere; 1e30: unbounded), from the TileSpan that culls the instance list.  Read only by the forward
// blend (blend.cu `reaches_rect`): each warp walks only the splats whose box meets its pixel rectangle.
struct __align__(16) SplatRec {
  float4 q0, q1, q2;
};
static_assert(sizeof(SplatRec) == 48, "SplatRec must be 48 bytes");

// Per-splat binning data (read by key emission and by preprocess-backward only): depth, 3-sigma radius, tile count.
struct __align__(16) SplatAux {
  float depth;
  int radius;
  uint32_t tiles;
  uint32_t pad;
};

// Per-splat 2-D gradient record accumulated by blend-backward (RED.ADD) and consumed by preprocess-backward:
//   (dL/dndc.x, dL/dndc.y, dL/dconic.xx, dL/dconic.xy, dL/dconic.yy, dL/dopacity, dL/dr, dL/dg, dL/db,
//    dL/dz (depth plane only; else pad), pad*2)
#define GAB_G2D_STRIDE 12

// The local viewer's export quantisation (GAB200_QUANTIZE_VIEWER): numpy's (np.clip(c, 0, 1) * 255).astype(np.uint8)
// on a float32 pixel, one rounded multiply and truncation.  fmaxf first: a NaN channel gives 0.
__device__ __forceinline__ uint32_t quantize_u8_viewer(float c) {
  return __float2uint_rz(__fmul_rn(fminf(fmaxf(c, 0.f), 1.f), 255.f));
}

struct Camera {  // staged once per block in shared memory
  float V[16];
  float Pm[16];
  float campos[3];
  float pad;
};

// carve helper: 256-B aligned sub-allocations inside a caller-provided byte buffer
struct Carver {
  char* base;
  size_t off;
  __host__ __device__ explicit Carver(void* p) : base(reinterpret_cast<char*>(p)), off(0) {}
  template <typename T>
  __host__ __device__ T* take(size_t count) {
    off = (off + 255) & ~size_t(255);
    T* r = reinterpret_cast<T*>(base + off);
    off += count * sizeof(T);
    return r;
  }
  __host__ __device__ size_t bytes() const { return (off + 255) & ~size_t(255); }
};

__host__ __device__ inline uint32_t tile_bits(uint32_t n) {  // bits needed for the tile id (reference: getHigherMsb)
  uint32_t msb = 16, step = 16;
  while (step > 1) {
    step /= 2;
    if (n >> msb)
      msb += step;
    else
      msb -= step;
  }
  if (n >> msb) msb++;
  return msb;
}

}  // namespace gab
