// composite.cu -- the capture loader's per-pixel RGBA composite on the device (gab200_composite_rgba).
//
// The reference's CameraDataset.__getitem__ (scene/__init__.py:48-51) turns a decoded RGBA frame into the (3,H,W)
// ground truth with numpy:
//     norm = rgba / 255.0;  arr = norm[..., :3] * norm[..., 3:4] + bg * (1 - norm[..., 3:4])
//     Image.fromarray(np.array(arr * 255.0, dtype=np.byte), "RGB")
// i.e. float64 arithmetic in that order, then a truncating cast (np.byte wraps on x86-64, and the bytes are read back
// as uint8), and the alpha channel is dropped.  Here every byte is the same double-precision expression, evaluated
// with explicitly rounded __ddiv_rn / __dmul_rn / __dsub_rn / __dadd_rn (no contraction into an FMA), then truncated:
// bit for bit the loader's bytes.  float32 in the same order gets 154 of the 65,536 (colour, alpha) pairs wrong on
// a black background and 391 on white; rounding instead of truncating gets about half of them wrong.
//
// The alpha byte itself goes to the mask plane (the foreground mask of GraphedFrame's mask term).
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

// loader byte of colour byte c over background bg at alpha unit value ua (= a / 255.0), om = 1 - ua
__device__ __forceinline__ uint8_t composite_byte(const double* __restrict__ unit, uint32_t c, double ua, double om,
                                                  double bg) {
  const double v = __dadd_rn(__dmul_rn(unit[c], ua), __dmul_rn(bg, om));
  return (uint8_t)__double2int_rz(__dmul_rn(v, 255.0));  // v * 255 lies in [0, 255 + 1e-13]: truncation
}

// One RGBA pixel (a little-endian word: R in the low byte) -> its three composite bytes and its alpha byte.
__device__ __forceinline__ void composite_px(const double* __restrict__ unit, uint32_t w, double b0, double b1,
                                             double b2, uint8_t& r, uint8_t& g, uint8_t& b, uint8_t& m) {
  const uint32_t a = w >> 24;
  const double ua = unit[a], om = __dsub_rn(1.0, ua);
  r = composite_byte(unit, w & 0xffu, ua, om, b0);
  g = composite_byte(unit, (w >> 8) & 0xffu, ua, om, b1);
  b = composite_byte(unit, (w >> 16) & 0xffu, ua, om, b2);
  m = (uint8_t)a;
}

// n = views * hw pixels.  Thread t takes pixels 4t .. 4t+3 of the flattened (views, H, W) grid.  VEC: hw % 4 == 0 (four
// pixels never straddle two views), rgba 16-B aligned, rgb / mask 4-B aligned (checked by the launcher): one 16-B load
// and one uchar4 store per plane.  Otherwise the scalar loop (ragged sizes, a view sliced out of a batch).
template <bool VEC>
__global__ void __launch_bounds__(256) composite_rgba_kernel(int64_t n, int64_t hw, const uint8_t* __restrict__ rgba,
                                                             const float* __restrict__ bg, uint8_t* __restrict__ rgb,
                                                             uint8_t* __restrict__ mask) {
  __shared__ double unit[256];  // k / 255.0, correctly rounded: the loader's `im_data / 255.0`
  unit[threadIdx.x] = __ddiv_rn((double)threadIdx.x, 255.0);
  const double b0 = (double)__ldg(bg), b1 = (double)__ldg(bg + 1), b2 = (double)__ldg(bg + 2);
  __syncthreads();
  const int64_t p4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (VEC && p4 + 3 < n) {
    const uint4 px = *reinterpret_cast<const uint4*>(rgba + p4 * 4);
    const int64_t k = p4 / hw, p = p4 - k * hw;
    uchar4 r, g, b, m;
    composite_px(unit, px.x, b0, b1, b2, r.x, g.x, b.x, m.x);
    composite_px(unit, px.y, b0, b1, b2, r.y, g.y, b.y, m.y);
    composite_px(unit, px.z, b0, b1, b2, r.z, g.z, b.z, m.z);
    composite_px(unit, px.w, b0, b1, b2, r.w, g.w, b.w, m.w);
    uint8_t* out = rgb + k * 3 * hw + p;
    *reinterpret_cast<uchar4*>(out) = r;
    *reinterpret_cast<uchar4*>(out + hw) = g;
    *reinterpret_cast<uchar4*>(out + 2 * hw) = b;
    if (mask != nullptr) *reinterpret_cast<uchar4*>(mask + k * hw + p) = m;
  } else {
    for (int64_t i = p4; i < n && i < p4 + 4; i++) {
      const uint8_t* q = rgba + i * 4;
      const uint32_t w = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
      const int64_t k = i / hw, p = i - k * hw;
      uint8_t r, g, b, m;
      composite_px(unit, w, b0, b1, b2, r, g, b, m);
      uint8_t* out = rgb + k * 3 * hw + p;
      out[0] = r;
      out[hw] = g;
      out[2 * hw] = b;
      if (mask != nullptr) mask[k * hw + p] = m;
    }
  }
}

void launch_composite_rgba(int64_t views, int H, int W, const uint8_t* rgba, const float* bg, uint8_t* rgb,
                           uint8_t* mask, cudaStream_t stream) {
  const int64_t hw = (int64_t)H * W, n = views * hw;
  if (n == 0) return;
  const unsigned blocks = (unsigned)(((n + 3) / 4 + 255) / 256);
  const bool aligned = hw % 4 == 0 && ((uintptr_t)rgba & 15) == 0 && (((uintptr_t)rgb | (uintptr_t)mask) & 3) == 0;
  if (aligned)
    composite_rgba_kernel<true><<<blocks, 256, 0, stream>>>(n, hw, rgba, bg, rgb, mask);
  else
    composite_rgba_kernel<false><<<blocks, 256, 0, stream>>>(n, hw, rgba, bg, rgb, mask);
  count_launch();
}

}  // namespace gab
