// metrics.cu -- forward-only image metrics of a render against its uint8 ground truth: mean L1, PSNR (two definitions)
// and mean SSIM of one view in two launches, with a deterministic reduction (include/gab200_rasterizer.h,
// gab200_image_metrics).  Replaces the evaluation of the reference's training_report (train.py:277-288: clamp, then
// l1_loss, psnr, ssim per val / test view) and of metrics.py:71-74 (ssim and psnr of the PNG bytes render.py wrote):
// one eager render plus ~40 launches of conv2d SSIM (utils/loss_utils.py:33-63) per view.
//
//   metrics_tile_kernel     : one 32x32 tile of one channel per CTA.  The SSIM statistics are those of
//                             ssim_stats_kernel (loss.cu): the same window, tile, zero padding and per-pixel formula,
//                             but no derivative map is written (there is no backward).  The CTA's sums of |d|, d^2
//                             and the SSIM map go to scratch, in double, at the CTA's index.
//   metrics_finalize_kernel : one CTA sums the partials in a fixed order (no floating-point atomics: the same inputs
//                             give the same bits on every call) and writes the view's record of four floats into row
//                             *row of the caller's table -- unless *skip_flag is set (an overflowed graph replay) or
//                             the row is out of range.
#include "common.cuh"
#include "kernels.cuh"
#include "ssim_tile.cuh"

namespace gab {

// SRC: GAB200_METRICS_FLOAT_CHW (float [3,H,W], clamped to [0, 1] as train.py:277 clamps it) or GAB200_METRICS_U8_HWC
// (the display image [H,W,3], value/255 as to_tensor reads render.py's PNG).  gt: uint8 [3,H,W].
template <int SRC>
__global__ void __launch_bounds__(256) metrics_tile_kernel(int H, int W, const void* __restrict__ render,
                                                           const uint8_t* __restrict__ gt, SsimWindow win,
                                                           double* __restrict__ partial) {
  __shared__ float sx[LIN][LIN + 1], sy[LIN][LIN + 1];
  __shared__ float hs[5][LIN][LT + 1];
  __shared__ double part[3][8];
  __shared__ GtFetch<uint8_t> fetch;
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT, ch = blockIdx.z;
  const int64_t plane = (int64_t)ch * H * W;
  fetch.init(tid);
  auto x_at = [&](int64_t px) -> float {   // px = y * W + x
    if constexpr (SRC == GAB200_METRICS_FLOAT_CHW) {
      const float v = static_cast<const float*>(render)[plane + px];
      return v != v ? v : fminf(fmaxf(v, 0.f), 1.f);   // torch.clamp(v, 0, 1): NaN stays NaN
    } else {
      return fetch.tab[static_cast<const uint8_t*>(render)[px * 3 + ch]];
    }
  };

  // tile + halo, one row per warp per round (zero outside the image: conv2d's padding)
#pragma unroll
  for (int rr = 0; rr < LROWS_PER_WARP; rr++) {
    const int r = wrp + rr * 8;
    if (r < LIN) {
      const int gy = y0 + r - LHALO;
      const bool row_ok = gy >= 0 && gy < H;
      const int64_t row = (int64_t)gy * W;
      const int gxa = x0 + lane - LHALO, gxb = gxa + 32;
      float xa = 0.f, ya = 0.f, xb = 0.f, yb = 0.f;
      if (row_ok && gxa >= 0 && gxa < W) {
        xa = x_at(row + gxa);
        ya = fetch(gt, plane + row + gxa);
      }
      if (lane < LIN - 32 && row_ok && gxb < W) {
        xb = x_at(row + gxb);
        yb = fetch(gt, plane + row + gxb);
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

  // horizontal pass: item = (row r, 8-column segment); mu1, mu2, E[x^2], E[y^2], E[xy]
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
  float l1_sum = 0.f, sq_sum = 0.f, ssim_sum = 0.f;
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
      ssim_sum += A1 * A2 * inv_b;
      const float d = sx[r0 + o + LHALO][col + LHALO] - sy[r0 + o + LHALO][col + LHALO];
      l1_sum += fabsf(d);
      sq_sum += d * d;
    }
  }
  // four pixels per thread in float, everything above in double
  double v[3] = {(double)l1_sum, (double)sq_sum, (double)ssim_sum};
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
#pragma unroll
    for (int q = 0; q < 3; q++) v[q] += __shfl_xor_sync(0xffffffffu, v[q], m);
  }
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 3; q++) part[q][wrp] = v[q];
  }
  __syncthreads();
  if (tid < 3) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < 8; w++) s += part[tid][w];
    const int64_t cta = ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[cta * 3 + tid] = s;   // channel-major: channel c's tiles are CTAs [c * tiles, (c + 1) * tiles)
  }
}

// One CTA: the 9 sums (3 channels x {|d|, d^2, SSIM}) over `tiles` partials each, in a fixed order, then the record
// {l1, psnr (mean of the per-channel PSNRs), psnr_all (one MSE over all values), ssim}.
__global__ void __launch_bounds__(256) metrics_finalize_kernel(int tiles, double inv_hw, double inv_n,
                                                               const double* __restrict__ partial,
                                                               const int32_t* __restrict__ row, int rows,
                                                               const int32_t* __restrict__ skip,
                                                               float* __restrict__ table) {
  if (skip != nullptr && *skip != 0) return;   // uniform over the CTA
  const int r = row != nullptr ? *row : 0;
  if (r < 0 || r >= rows) return;
  __shared__ double part[9][8];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  double v[9];
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const int c = k / 3, q = k - 3 * (k / 3);
    double s = 0.0;
    for (int i = tid; i < tiles; i += 256) s += partial[((int64_t)c * tiles + i) * 3 + q];
    v[k] = s;
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
#pragma unroll
    for (int k = 0; k < 9; k++) v[k] += __shfl_xor_sync(0xffffffffu, v[k], m);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 9; k++) part[k][wrp] = v[k];
  }
  __syncthreads();
  if (tid == 0) {
    double S[9];
#pragma unroll
    for (int k = 0; k < 9; k++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++) s += part[k][w];
      S[k] = s;
    }
    // 20 log10(1 / sqrt(MSE)) = -10 log10(MSE); an MSE of 0 gives +inf, as torch does
    double psnr = 0.0;
#pragma unroll
    for (int c = 0; c < 3; c++) psnr += -10.0 * log10(S[3 * c + 1] * inv_hw);
    float* rec = table + (int64_t)r * GAB200_METRICS_FIELDS;
    rec[0] = (float)((S[0] + S[3] + S[6]) * inv_n);
    rec[1] = (float)(psnr * (1.0 / 3.0));
    rec[2] = (float)(-10.0 * log10((S[1] + S[4] + S[7]) * inv_n));
    rec[3] = (float)((S[2] + S[5] + S[8]) * inv_n);
  }
}

static int metrics_tiles(int H, int W) { return ((W + LT - 1) / LT) * ((H + LT - 1) / LT); }

size_t metrics_scratch_bytes(int H, int W) { return (size_t)metrics_tiles(H, W) * 3 * 3 * sizeof(double); }

void launch_image_metrics(int H, int W, int kind, const void* render, const uint8_t* gt, const int32_t* row, int rows,
                          const int32_t* skip, float* table, void* scratch, cudaStream_t stream) {
  const SsimWindow win = ssim_window();
  const dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, 3);
  double* partial = static_cast<double*>(scratch);
  if (kind == GAB200_METRICS_FLOAT_CHW)
    metrics_tile_kernel<GAB200_METRICS_FLOAT_CHW><<<grid, 256, 0, stream>>>(H, W, render, gt, win, partial);
  else
    metrics_tile_kernel<GAB200_METRICS_U8_HWC><<<grid, 256, 0, stream>>>(H, W, render, gt, win, partial);
  count_launch();
  const double hw = (double)H * W;   // the means multiply by reciprocals formed here: no division on the device
  metrics_finalize_kernel<<<1, 256, 0, stream>>>(metrics_tiles(H, W), 1.0 / hw, 1.0 / (3.0 * hw), partial, row, rows,
                                                 skip, table);
  count_launch();
}

}  // namespace gab
