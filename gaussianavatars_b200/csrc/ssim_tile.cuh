// ssim_tile.cuh -- the separable 11x11 SSIM tile machinery shared by the training loss (loss.cu: ssim_stats_kernel,
// ssim_grad_kernel) and the forward-only image metrics (metrics.cu): the tile geometry, the Gaussian window of
// utils/loss_utils.py:23-25, the 11-tap register pass and the correctly rounded uint8 -> [0, 1] conversion.
#pragma once

#include <cmath>
#include <cstdint>

namespace gab {

constexpr int LT = 32;             // tile edge (outputs)
constexpr int LHALO = 5;           // window_size // 2
constexpr int LIN = LT + 2 * LHALO;
constexpr int LTAPS = 2 * LHALO + 1;
constexpr int LSEG_H = 8;          // outputs per thread, horizontal pass (168 work items per tile)
constexpr int LLOAD_H = LSEG_H + LTAPS - 1;
constexpr int LSEG = 4;            // outputs per thread, vertical pass (256 work items per tile)
constexpr int LLOAD = LSEG + LTAPS - 1;
constexpr int LROWS_PER_WARP = (LIN + 7) / 8;

struct SsimWindow { float w[LTAPS]; };

// gaussian(11, 1.5) of utils/loss_utils.py:23-25, in float like the reference's torch.Tensor (the float32 taps are
// summed in double and rounded once: that reproduces torch.Tensor.sum()'s value)
inline SsimWindow ssim_window() {
  SsimWindow win;
  float g[LTAPS];
  double sum = 0.0;
  for (int i = 0; i < LTAPS; i++) {
    g[i] = (float)exp(-(double)((i - LHALO) * (i - LHALO)) / (2.0 * 1.5 * 1.5));
    sum += (double)g[i];
  }
  for (int i = 0; i < LTAPS; i++) win.w[i] = g[i] / (float)sum;
  return win;
}

// value / 255 with a correctly rounded division: bit-identical to the reference's CPU-side
// `torch.from_numpy(np.array(img)) / 255.0` (utils/general_utils.py:21-23); a multiply by 1/255 is off by one ulp
// for some codes and flips sign(x - y).  The tile kernels divide once per code into a 256-entry shared table.
__device__ __forceinline__ float u8_unit(uint8_t v) { return __fdiv_rn((float)v, 255.f); }

template <typename GT> struct GtFetch;
template <> struct GtFetch<uint8_t> {
  float tab[256];
  __device__ __forceinline__ void init(int tid) {
    tab[tid] = u8_unit((uint8_t)tid);  // blockDim.x == 256
    __syncthreads();
  }
  __device__ __forceinline__ float operator()(const uint8_t* p, int64_t i) const { return tab[p[i]]; }
};
template <> struct GtFetch<float> {
  __device__ __forceinline__ void init(int) {}
  __device__ __forceinline__ float operator()(const float* p, int64_t i) const { return p[i]; }
};

// 11-tap pass over a register window: out[o] = sum_t w[t] v[o + t]
template <int NOUT>
__device__ __forceinline__ void taps(const SsimWindow& win, const float (&v)[NOUT + LTAPS - 1], float (&out)[NOUT]) {
#pragma unroll
  for (int o = 0; o < NOUT; o++) {
    float a = 0.f;
#pragma unroll
    for (int t = 0; t < LTAPS; t++) a = fmaf(win.w[t], v[o + t], a);
    out[o] = a;
  }
}

}  // namespace gab
