// loss.cu -- L1 photometric loss against a uint8 ground-truth image, forward and gradient in ONE pass over the
// rendered image (SURVEY.md 8f rank 2, the first half of train.py:128-131: `gt_image.cuda()`, `l1_loss(image, gt)`).
// The reference uploads the ground truth as float32 (4 B/px/channel) and runs ~6 eager kernels for L1 + its autograd;
// here the uint8 image is uploaded (1 B), converted in-register, and dL/dimage = sign(render - gt) / n is written in the
// same kernel that accumulates the loss.
#include "common.cuh"
#include "kernels.cuh"
#include "ssim_tile.cuh"

namespace gab {

// VEC: img/grad 16-B aligned and gt 4-B aligned (checked by the launcher); otherwise every thread takes the scalar loop.
// grad == nullptr: loss only.  loss_sum == nullptr: gradient only.  upstream (device scalar, may be NULL = 1) scales the
// gradient: the backward of `loss = l1(img, gt)` under autograd is this kernel with loss_sum == nullptr, so no separate
// multiply pass over the (3,H,W) gradient is needed.
template <bool VEC>
__global__ void __launch_bounds__(256) l1_loss_u8_kernel(int64_t n, const float* __restrict__ img,
                                                         const uint8_t* __restrict__ gt, float inv_n_,
                                                         const float* __restrict__ upstream,
                                                         float* __restrict__ grad, float* __restrict__ loss_sum) {
  const int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const float inv_n = upstream != nullptr ? inv_n_ * __ldg(upstream) : inv_n_;
  float acc = 0.f;
  if (VEC && i4 + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(img + i4);
    const uchar4 g = *reinterpret_cast<const uchar4*>(gt + i4);
    const float d0 = v.x - __fdiv_rn((float)g.x, 255.f), d1 = v.y - __fdiv_rn((float)g.y, 255.f);
    const float d2 = v.z - __fdiv_rn((float)g.z, 255.f), d3 = v.w - __fdiv_rn((float)g.w, 255.f);
    acc = fabsf(d0) + fabsf(d1) + fabsf(d2) + fabsf(d3);
    auto sgn = [](float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f); };
    if (grad != nullptr)
      *reinterpret_cast<float4*>(grad + i4) = make_float4(sgn(d0) * inv_n, sgn(d1) * inv_n, sgn(d2) * inv_n, sgn(d3) * inv_n);
  } else {
    for (int64_t i = i4; i < n && i < i4 + 4; i++) {
      const float d = img[i] - __fdiv_rn((float)gt[i], 255.f);
      acc += fabsf(d);
      if (grad != nullptr) grad[i] = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * inv_n;
    }
  }
  if (loss_sum == nullptr) return;  // gradient-only launch (uniform: no barrier is skipped by part of a block)
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) s += part[w];
    atomicAdd(loss_sum, s * inv_n_);
  }
}

void launch_l1_loss_u8(int64_t n, const float* img, const uint8_t* gt, const float* upstream, float* grad, float* loss,
                       cudaStream_t stream) {
  if (n == 0) return;
  const int64_t threads = (n + 3) / 4;
  const bool aligned = (((uintptr_t)img | (uintptr_t)grad) & 15) == 0 && ((uintptr_t)gt & 3) == 0;
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  if (aligned)
    l1_loss_u8_kernel<true><<<blocks, 256, 0, stream>>>(n, img, gt, 1.0f / (float)n, upstream, grad, loss);
  else  // a contiguous view with a storage offset (batch[b], a uint8 slice): same result through scalar accesses
    l1_loss_u8_kernel<false><<<blocks, 256, 0, stream>>>(n, img, gt, 1.0f / (float)n, upstream, grad, loss);
  count_launch();
}

// ================================================================================================================
// Photometric training loss  (1 - lambda) * L1 + lambda * (1 - SSIM)  with its gradient   (SURVEY.md 8f rank 2)
// ================================================================================================================
// The reference evaluates SSIM with five grouped 11x11 convolutions and lets autograd run five more backwards
// (utils/loss_utils.py:36-63, train.py:131-132): ~40 eager launches and ten (3,H,W) temporaries per step.  Here it is
// two launches.  The Gaussian window is separable, so every 32x32 tile does an 11-tap horizontal pass out of a
// 42x42 shared-memory tile and an 11-tap vertical pass out of the result, register-blocked (a thread produces eight
// horizontal outputs from 18 loaded values, four vertical outputs from 14).
//
//   ssim_stats_kernel : mu1, mu2, E[x^2], E[y^2], E[xy]  ->  the SSIM map (summed into loss[1]) and the three partial
//                       derivatives  ds/dmu1, ds/dE[x^2], ds/dE[xy]  per pixel (12 B/px/channel of scratch);
//                       the L1 term is summed in the same pass (loss[0]).
//   ssim_grad_kernel  : d(sum_p s(p))/dx(q) = (G * ds/dmu1)(q) + 2 x(q) (G * ds/dE[x^2])(q) + y(q) (G * ds/dE[xy])(q)
//                       (G symmetric, zero padding on both sides as conv2d(padding=5) does), combined with the L1
//                       sign term into dL/dimage; the launch also writes loss[2] = the total.
//
// With s = A1 A2 / (B1 B2),  A1 = 2 mu1 mu2 + C1,  A2 = 2 (E[xy] - mu1 mu2) + C2,  B1 = mu1^2 + mu2^2 + C1,
// B2 = E[x^2] - mu1^2 + E[y^2] - mu2^2 + C2:
//   ds/dmu1    = 2 mu2 (A2 - A1) / (B1 B2) - 2 mu1 A1 A2 (B2 - B1) / (B1 B2)^2
//   ds/dE[x^2] = -A1 A2 / (B1 B2^2)
//   ds/dE[xy]  = 2 A1 / (B1 B2)

// The tile geometry (LT, LHALO, ...), SsimWindow, u8_unit, GtFetch and taps live in ssim_tile.cuh, shared with the
// forward-only image metrics (metrics.cu).

template <typename GT>
__global__ void __launch_bounds__(256) ssim_stats_kernel(int H, int W, const float* __restrict__ img,
                                                         const GT* __restrict__ gt, SsimWindow win,
                                                         float* __restrict__ maps, int64_t map_stride,
                                                         double* __restrict__ sums) {
  __shared__ float sx[LIN][LIN + 1], sy[LIN][LIN + 1];
  __shared__ float hs[5][LIN][LT + 1];
  __shared__ float part[2][8];
  __shared__ GtFetch<GT> fetch;
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
  const int64_t plane = (int64_t)blockIdx.z * H * W;
  fetch.init(tid);

  // tile + halo, one row per warp per round (zero outside the image: conv2d's padding)
#pragma unroll
  for (int rr = 0; rr < LROWS_PER_WARP; rr++) {
    const int r = wrp + rr * 8;
    if (r < LIN) {
      const int gy = y0 + r - LHALO;
      const bool row_ok = gy >= 0 && gy < H;
      const int64_t row = plane + (int64_t)gy * W;
      const int gxa = x0 + lane - LHALO, gxb = gxa + 32;
      float xa = 0.f, ya = 0.f, xb = 0.f, yb = 0.f;
      if (row_ok && gxa >= 0 && gxa < W) {
        xa = img[row + gxa];
        ya = fetch(gt, row + gxa);
      }
      if (lane < LIN - 32 && row_ok && gxb < W) {
        xb = img[row + gxb];
        yb = fetch(gt, row + gxb);
      }
      sx[r][lane] = xa;
      sy[r][lane] = ya;
      if (lane < LIN - 32) {
        sx[r][32 + lane] = xb;
        sy[r][32 + lane] = yb;
      }
    }
  }
  __syncthreads();

  // horizontal pass: item = (row r, 8-column segment); consecutive lanes take consecutive rows (stride 43: no conflicts)
  if (tid < LIN * (LT / LSEG_H)) {
    const int seg = tid / LIN, r = tid - seg * LIN;
    const int c0 = seg * LSEG_H;
    float xv[LLOAD_H], yv[LLOAD_H], pv[LLOAD_H], out[LSEG_H];
#pragma unroll
    for (int k = 0; k < LLOAD_H; k++) {
      xv[k] = sx[r][c0 + k];
      yv[k] = sy[r][c0 + k];
    }
    taps<LSEG_H>(win, xv, out);
#pragma unroll
    for (int o = 0; o < LSEG_H; o++) hs[0][r][c0 + o] = out[o];
    taps<LSEG_H>(win, yv, out);
#pragma unroll
    for (int o = 0; o < LSEG_H; o++) hs[1][r][c0 + o] = out[o];
#pragma unroll
    for (int k = 0; k < LLOAD_H; k++) pv[k] = xv[k] * xv[k];
    taps<LSEG_H>(win, pv, out);
#pragma unroll
    for (int o = 0; o < LSEG_H; o++) hs[2][r][c0 + o] = out[o];
#pragma unroll
    for (int k = 0; k < LLOAD_H; k++) pv[k] = yv[k] * yv[k];
    taps<LSEG_H>(win, pv, out);
#pragma unroll
    for (int o = 0; o < LSEG_H; o++) hs[3][r][c0 + o] = out[o];
#pragma unroll
    for (int k = 0; k < LLOAD_H; k++) pv[k] = xv[k] * yv[k];
    taps<LSEG_H>(win, pv, out);
#pragma unroll
    for (int o = 0; o < LSEG_H; o++) hs[4][r][c0 + o] = out[o];
  }
  __syncthreads();

  // vertical pass: thread = (column, group of 4 rows)
  const int col = lane, r0 = wrp * LSEG;
  float out[5][LSEG];
#pragma unroll
  for (int q = 0; q < 5; q++) {
    float v[LLOAD];
#pragma unroll
    for (int k = 0; k < LLOAD; k++) v[k] = hs[q][r0 + k][col];
    taps<LSEG>(win, v, out[q]);
  }
  const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
  float l1_sum = 0.f, ssim_sum = 0.f;
  const int gx = x0 + col;
#pragma unroll
  for (int o = 0; o < LSEG; o++) {
    const int gy = y0 + r0 + o;
    if (gx < W && gy < H) {
      const float mu1 = out[0][o], mu2 = out[1][o];
      const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
      const float s1 = out[2][o] - mu1_sq, s2 = out[3][o] - mu2_sq, s12 = out[4][o] - mu12;
      const float A1 = 2.f * mu12 + C1, A2 = 2.f * s12 + C2;
      const float B1 = mu1_sq + mu2_sq + C1, B2 = s1 + s2 + C2;
      const float inv_b = 1.f / (B1 * B2);
      const float s = A1 * A2 * inv_b;
      const float d_mu1 = 2.f * mu2 * (A2 - A1) * inv_b - 2.f * mu1 * s * (B2 - B1) * inv_b;
      const float d_ex2 = -s * (B1 * inv_b);  // -s / B2
      const float d_exy = 2.f * A1 * inv_b;
      const int64_t o_px = plane + (int64_t)gy * W + gx;
      maps[o_px] = d_mu1;
      maps[map_stride + o_px] = d_ex2;
      maps[2 * map_stride + o_px] = d_exy;
      ssim_sum += s;
      l1_sum += fabsf(sx[r0 + o + LHALO][col + LHALO] - sy[r0 + o + LHALO][col + LHALO]);
    }
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
    l1_sum += __shfl_xor_sync(0xffffffffu, l1_sum, m);
    ssim_sum += __shfl_xor_sync(0xffffffffu, ssim_sum, m);
  }
  if (lane == 0) {
    part[0][wrp] = l1_sum;
    part[1][wrp] = ssim_sum;
  }
  __syncthreads();
  if (tid < 2) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) s += part[tid][w];
    atomicAdd(sums + tid, (double)s);  // ~10^3 block sums of up to 1024 terms each: float atomics would cost 1e-6
  }
}

template <typename GT>
__global__ void __launch_bounds__(256) ssim_grad_kernel(int H, int W, const float* __restrict__ img,
                                                        const GT* __restrict__ gt, SsimWindow win, float inv_n,
                                                        float lambda, const float* __restrict__ maps,
                                                        int64_t map_stride, float* __restrict__ grad,
                                                        const double* __restrict__ sums, float* __restrict__ loss) {
  __shared__ float sm[3][LIN][LIN + 1];
  __shared__ float hs[3][LIN][LT + 1];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  // reverse of the stats kernel's block order: the maps it wrote last are the ones still in L2
  const int x0 = (gridDim.x - 1 - blockIdx.x) * LT, y0 = (gridDim.y - 1 - blockIdx.y) * LT;
  const int ch = gridDim.z - 1 - blockIdx.z;
  const int64_t plane = (int64_t)ch * H * W;

#pragma unroll
  for (int rr = 0; rr < LROWS_PER_WARP; rr++) {
    const int r = wrp + rr * 8;
    if (r < LIN) {
      const int gy = y0 + r - LHALO;
      const bool row_ok = gy >= 0 && gy < H;
      const int64_t row = plane + (int64_t)gy * W;
      const int gxa = x0 + lane - LHALO, gxb = gxa + 32;
      const bool oka = row_ok && gxa >= 0 && gxa < W, okb = lane < LIN - 32 && row_ok && gxb < W;
      float a[3] = {0.f, 0.f, 0.f}, b[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int q = 0; q < 3; q++) {
        if (oka) a[q] = maps[q * map_stride + row + gxa];
        if (okb) b[q] = maps[q * map_stride + row + gxb];
      }
#pragma unroll
      for (int q = 0; q < 3; q++) {
        sm[q][r][lane] = a[q];
        if (lane < LIN - 32) sm[q][r][32 + lane] = b[q];
      }
    }
  }
  __syncthreads();
  if (tid < LIN * (LT / LSEG_H)) {
    const int seg = tid / LIN, r = tid - seg * LIN;
    const int c0 = seg * LSEG_H;
#pragma unroll
    for (int q = 0; q < 3; q++) {
      float v[LLOAD_H], out[LSEG_H];
#pragma unroll
      for (int k = 0; k < LLOAD_H; k++) v[k] = sm[q][r][c0 + k];
      taps<LSEG_H>(win, v, out);
#pragma unroll
      for (int o = 0; o < LSEG_H; o++) hs[q][r][c0 + o] = out[o];
    }
  }
  __syncthreads();
  const int col = lane, r0 = wrp * LSEG;
  float out[3][LSEG];
#pragma unroll
  for (int q = 0; q < 3; q++) {
    float v[LLOAD];
#pragma unroll
    for (int k = 0; k < LLOAD; k++) v[k] = hs[q][r0 + k][col];
    taps<LSEG>(win, v, out[q]);
  }
  const int gx = x0 + col;
  const float k_l1 = (1.f - lambda) * inv_n, k_ssim = -lambda * inv_n;
#pragma unroll
  for (int o = 0; o < LSEG; o++) {
    const int gy = y0 + r0 + o;
    if (gx < W && gy < H) {
      const int64_t o_px = plane + (int64_t)gy * W + gx;
      const float x = img[o_px];
      float y;
      if constexpr (sizeof(GT) == 1) y = u8_unit(gt[o_px]); else y = gt[o_px];
      const float d = x - y;
      const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
      const float dssim = out[0][o] + 2.f * x * out[1][o] + y * out[2][o];
      grad[o_px] = k_l1 * sgn + k_ssim * dssim;
    }
  }
  // the stats kernel has completed (stream order): fold its two sums into the three reported means
  if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && tid == 0) {
    const double l1 = sums[0] * (double)inv_n, ssim = sums[1] * (double)inv_n;
    loss[0] = (float)l1;
    loss[1] = (float)ssim;
    loss[2] = (float)((1.0 - (double)lambda) * l1 + (double)lambda * (1.0 - ssim));
  }
}

template <typename GT>
static void launch_photometric_t(int C, int H, int W, const float* img, const GT* gt, float lambda, float* grad,
                                 float* loss, float* scratch, cudaStream_t stream) {
  const SsimWindow win = ssim_window();
  const int64_t n = (int64_t)C * H * W;
  const dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, C);
  double* sums = reinterpret_cast<double*>(scratch);  // [2], zeroed by the caller (api.cu); the maps follow
  float* maps = scratch + GAB_PHOTOMETRIC_SCRATCH_HEAD;
  ssim_stats_kernel<GT><<<grid, 256, 0, stream>>>(H, W, img, gt, win, maps, n, sums);
  count_launch();
  ssim_grad_kernel<GT><<<grid, 256, 0, stream>>>(H, W, img, gt, win, 1.0f / (float)n, lambda, maps, n, grad, sums, loss);
  count_launch();
}

void launch_photometric_loss(int C, int H, int W, const float* img, const void* gt, int gt_is_u8, float lambda,
                             float* grad, float* loss, float* scratch, cudaStream_t stream) {
  if ((int64_t)C * H * W == 0) return;
  if (gt_is_u8)
    launch_photometric_t<uint8_t>(C, H, W, img, (const uint8_t*)gt, lambda, grad, loss, scratch, stream);
  else
    launch_photometric_t<float>(C, H, W, img, (const float*)gt, lambda, grad, loss, scratch, stream);
}

}  // namespace gab
