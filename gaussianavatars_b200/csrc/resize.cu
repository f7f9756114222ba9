// resize.cu -- Pillow's bicubic resize of 8-bit planes on the device (gab200_resize_u8).
//
// The reference's loader resizes every composited frame to its camera's size with PIL's `image.resize(size)`
// (PILtoTorch, utils/general_utils.py:21-22): the default BICUBIC filter of an "RGB" image.  That resize is exact
// integer arithmetic on weights made in double precision, so it is restated here bit for bit (oracle/resize.py holds
// the same algorithm in numpy and the rule it follows):
//
//   plan        one thread per output column and row: the axis' first input, tap count and 22-bit fixed-point weights,
//               every double operation explicitly rounded (__dmul_rn / __dadd_rn / ...: no contraction into an FMA),
//               so the tables are those of the host's C double arithmetic.  Sizes only: no host work, no upload.
//   horizontal  one CTA per (plane, input row), the row staged in shared memory: out_w bytes, each the int32 sum from
//               2^21 of pixel * weight, >> 22 and clamped -- into a uint8 intermediate, or straight into dst when the
//               height does not change.
//   vertical    one CTA per (plane, output row), threads along x (coalesced), the row's weights broadcast: reads the
//               intermediate (or src when the width does not change) and writes dst.
//
// An axis whose size does not change is not resampled (as in Pillow); when neither changes dst is a copy of src.
// Nothing is allocated and nothing is read on the host: the call can be captured in a graph.
#include "common.cuh"
#include "kernels.cuh"

namespace gab {
namespace {

constexpr int RESIZE_THREADS = 256;
constexpr int RESIZE_PRECISION = 22;
constexpr int RESIZE_STAGE_MAX = 48 * 1024;   // a wider input row is read from global memory instead of staged

struct ResizeAxis {
  int in, out, ksize;   // ksize = 0: the axis is not resampled
};

ResizeAxis resize_axis(int in, int out) {
  if (in == out) return {in, out, 0};
  const double scale = (double)in / (double)out;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  return {in, out, (int)ceil(2.0 * filterscale) * 2 + 1};
}

struct ResizeScratch {
  int2* hbounds;
  int32_t* hcoef;
  int2* vbounds;
  int32_t* vcoef;
  uint8_t* tmp;
};

// The scratch: each resampled axis' bounds and weights, and the intermediate when both axes are resampled.
ResizeScratch carve_resize(Carver& c, int64_t planes, const ResizeAxis& h, const ResizeAxis& v) {
  ResizeScratch s;
  s.hbounds = c.take<int2>(h.ksize ? h.out : 0);
  s.hcoef = c.take<int32_t>(h.ksize ? (size_t)h.out * h.ksize : 0);
  s.vbounds = c.take<int2>(v.ksize ? v.out : 0);
  s.vcoef = c.take<int32_t>(v.ksize ? (size_t)v.out * v.ksize : 0);
  s.tmp = c.take<uint8_t>(h.ksize && v.ksize ? (size_t)planes * v.in * h.out : 0);
  return s;
}

// The Keys cubic, a = -0.5: (1.5 t - 2.5) t t + 1 on |t| < 1, (((t - 5) t + 8) t - 4) * -0.5 on |t| < 2.
__device__ double bicubic(double t) {
  t = fabs(t);
  if (t < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, t), 2.5), t), t), 1.0);
  if (t < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(t, 5.0), t), 8.0), t), 4.0), -0.5);
  return 0.0;
}

// Output index i of an axis in -> out: bounds (first input, taps) and ksize weights (0 past the taps).
__device__ void plan_index(int i, int in, int out, int ksize, int2* __restrict__ bounds, int32_t* __restrict__ coef) {
  const double scale = __ddiv_rn((double)in, (double)out);
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(2.0, filterscale);
  const double ss = __ddiv_rn(1.0, filterscale);
  const double center = __dmul_rn(__dadd_rn((double)i, 0.5), scale);
  const int first = max(__double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5)), 0);
  const int last = min(__double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5)), in);
  const int taps = min(max(last - first, 0), ksize);
  double sum = 0.0;
  for (int j = 0; j < taps; j++)
    sum = __dadd_rn(sum, bicubic(__dmul_rn(__dadd_rn(__dsub_rn((double)(j + first), center), 0.5), ss)));
  int32_t* k = coef + (size_t)i * ksize;
  for (int j = 0; j < ksize; j++) {
    int32_t q = 0;
    if (j < taps) {
      double w = bicubic(__dmul_rn(__dadd_rn(__dsub_rn((double)(j + first), center), 0.5), ss));
      if (sum != 0.0) w = __ddiv_rn(w, sum);
      q = __double2int_rz(__dadd_rn(__dmul_rn(w, (double)(1 << RESIZE_PRECISION)), w < 0.0 ? -0.5 : 0.5));
    }
    k[j] = q;
  }
  bounds[i] = make_int2(first, taps);
}

__global__ void __launch_bounds__(RESIZE_THREADS) resize_plan_kernel(ResizeAxis h, ResizeAxis v, ResizeScratch s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int nh = h.ksize ? h.out : 0, nv = v.ksize ? v.out : 0;
  if (i < nh)
    plan_index(i, h.in, h.out, h.ksize, s.hbounds, s.hcoef);
  else if (i < nh + nv)
    plan_index(i - nh, v.in, v.out, v.ksize, s.vbounds, s.vcoef);
}

__device__ __forceinline__ uint8_t clip8(int32_t acc) {
  return (uint8_t)min(max(acc >> RESIZE_PRECISION, 0), 255);
}

// One CTA per input row of every plane (blockIdx.x = plane * in_h + y): row -> out_w bytes of dst's row.
template <bool kStaged>
__global__ void __launch_bounds__(RESIZE_THREADS) resize_horizontal_kernel(int in_w, int out_w, int ksize,
                                                                           const uint8_t* __restrict__ src,
                                                                           const int2* __restrict__ bounds,
                                                                           const int32_t* __restrict__ coef,
                                                                           uint8_t* __restrict__ dst) {
  extern __shared__ uint8_t stage[];
  const uint8_t* row = src + (int64_t)blockIdx.x * in_w;
  if (kStaged) {
    for (int x = threadIdx.x; x < in_w; x += RESIZE_THREADS) stage[x] = row[x];
    __syncthreads();
  }
  const uint8_t* in = kStaged ? stage : row;
  uint8_t* out = dst + (int64_t)blockIdx.x * out_w;
  for (int xx = threadIdx.x; xx < out_w; xx += RESIZE_THREADS) {
    const int2 b = bounds[xx];
    const int32_t* k = coef + (size_t)xx * ksize;
    int32_t acc = 1 << (RESIZE_PRECISION - 1);
    for (int j = 0; j < b.y; j++) acc += (int32_t)in[b.x + j] * k[j];
    out[xx] = clip8(acc);
  }
}

// One CTA per output row of every plane (blockIdx.x = plane * out_h + yy), threads along x.
__global__ void __launch_bounds__(RESIZE_THREADS) resize_vertical_kernel(int in_h, int out_h, int w, int ksize,
                                                                         const uint8_t* __restrict__ src,
                                                                         const int2* __restrict__ bounds,
                                                                         const int32_t* __restrict__ coef,
                                                                         uint8_t* __restrict__ dst) {
  const int64_t plane = blockIdx.x / out_h;
  const int yy = blockIdx.x - (int)(plane * out_h);
  const int2 b = bounds[yy];
  const int32_t* k = coef + (size_t)yy * ksize;
  const uint8_t* in = src + (plane * in_h + b.x) * w;
  uint8_t* out = dst + (int64_t)blockIdx.x * w;
  for (int xx = threadIdx.x; xx < w; xx += RESIZE_THREADS) {
    int32_t acc = 1 << (RESIZE_PRECISION - 1);
    for (int j = 0; j < b.y; j++) acc += (int32_t)in[(int64_t)j * w + xx] * k[j];
    out[xx] = clip8(acc);
  }
}

}  // namespace

size_t resize_scratch_bytes(int64_t planes, int in_h, int in_w, int out_h, int out_w) {
  if (planes <= 0 || in_h <= 0 || in_w <= 0 || out_h <= 0 || out_w <= 0) return 0;
  if (planes * in_h > INT32_MAX || planes * out_h > INT32_MAX) return 0;   // one CTA per row of every plane
  Carver c(nullptr);
  carve_resize(c, planes, resize_axis(in_w, out_w), resize_axis(in_h, out_h));
  return c.bytes() == 0 ? 256 : c.bytes();   // a same-size copy still takes a (unused) non-empty scratch
}

void launch_resize_u8(int64_t planes, int in_h, int in_w, int out_h, int out_w, const uint8_t* src, uint8_t* dst,
                      void* scratch, cudaStream_t stream) {
  const ResizeAxis h = resize_axis(in_w, out_w), v = resize_axis(in_h, out_h);
  if (!h.ksize && !v.ksize) {
    cudaMemcpyAsync(dst, src, (size_t)planes * in_h * in_w, cudaMemcpyDeviceToDevice, stream);
    return;
  }
  Carver c(scratch);
  const ResizeScratch s = carve_resize(c, planes, h, v);
  const int n_plan = (h.ksize ? h.out : 0) + (v.ksize ? v.out : 0);
  resize_plan_kernel<<<(n_plan + RESIZE_THREADS - 1) / RESIZE_THREADS, RESIZE_THREADS, 0, stream>>>(h, v, s);
  if (h.ksize) {
    uint8_t* hout = v.ksize ? s.tmp : dst;
    const unsigned rows = (unsigned)(planes * in_h);
    if (in_w <= RESIZE_STAGE_MAX)
      resize_horizontal_kernel<true><<<rows, RESIZE_THREADS, in_w, stream>>>(in_w, out_w, h.ksize, src, s.hbounds,
                                                                            s.hcoef, hout);
    else
      resize_horizontal_kernel<false><<<rows, RESIZE_THREADS, 0, stream>>>(in_w, out_w, h.ksize, src, s.hbounds,
                                                                          s.hcoef, hout);
  }
  if (v.ksize)
    resize_vertical_kernel<<<(unsigned)(planes * out_h), RESIZE_THREADS, 0, stream>>>(
        in_h, out_h, out_w, v.ksize, h.ksize ? s.tmp : src, s.vbounds, s.vcoef, dst);
}

}  // namespace gab
