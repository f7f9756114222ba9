// lpips.cu -- forward-only LPIPS distance (v0.1, AlexNet or VGG-16 features) of one rendered view against its uint8
// ground truth, with no host wait (include/gab200_rasterizer.h, gab200_lpips).  Replaces lpipsPyTorch's LPIPS as
// train.py's training_report (AlexNet) and metrics.py (VGG-16) call it: z-score, torchvision `features` up to the
// last target ReLU, per target layer the channel-normalised squared difference weighted by the lin layer and averaged
// over the pixels, summed over the five layers.
//
//   lpips_input_kernel    : both images -> z-scored fp32 NHWC activations, 4 channels (the 4th is 0, so the first
//                           convolution gathers one float4 per tap like every other layer).
//   lpips_conv_kernel     : convolution + bias + ReLU as an implicit GEMM on the tensor cores (mma.sync m16n8k8,
//                           TF32 operands rounded to nearest with cvt.rna, FP32 accumulation).  M = output pixels of
//                           both images, N = Cout, K = (ky, kx, ci) padded to BK.  One template over (k, stride, pad);
//                           the K loop runs in one fixed order and there is no split-K, so every output has a fixed
//                           summation order.
//   lpips_pool_kernel     : max pool, floor sizes, exact.
//   lpips_head_kernel     : at a target layer, per pixel the two channel norms, the normalised squared difference and
//                           the lin dot product in FP32; each CTA's sum over its pixels goes to scratch in double at
//                           the CTA's index.
//   lpips_finalize_kernel : one CTA adds the partials in a fixed order, forms each layer's mean and the sum over the
//                           layers, and writes one float into row *row of the caller's table (nothing when *skip_flag).
// No floating-point atomics anywhere: the same inputs and weights give the same bits on every call.
//
// Packed weights (gab200_lpips_pack; this file alone knows the layout): per convolution, W as [Kpad][Cout] floats
// already rounded to TF32 (k = (ky * ks + kx) * Cs + ci, Cs = 4 for the RGB layer, zero rows past ks * ks * Cs or
// ci >= Cin), then the Cout biases in FP32; after the last convolution the five lin weight vectors.
#include "common.cuh"
#include "kernels.cuh"
#include "ssim_tile.cuh"

namespace gab {

namespace {

struct LpConv {
  int cin, cout, ks, stride, pad;
  bool pool_after, target;
};
struct LpNet {
  int nconv, pool_k;
  LpConv conv[13];
};

// torchvision alexnet().features / vgg16().features up to the last target ReLU (lpipsPyTorch's target_layers: the
// ReLU before each pool, and the last one).  The pools are 3x3 stride 2 (AlexNet) and 2x2 stride 2 (VGG-16).
const LpNet kAlex = {5, 3, {{3, 64, 11, 4, 2, true, true}, {64, 192, 5, 1, 2, true, true},
                            {192, 384, 3, 1, 1, false, true}, {384, 256, 3, 1, 1, false, true},
                            {256, 256, 3, 1, 1, false, true}}};
const LpNet kVgg = {13, 2, {{3, 64, 3, 1, 1, false, false}, {64, 64, 3, 1, 1, true, true},
                            {64, 128, 3, 1, 1, false, false}, {128, 128, 3, 1, 1, true, true},
                            {128, 256, 3, 1, 1, false, false}, {256, 256, 3, 1, 1, false, false},
                            {256, 256, 3, 1, 1, true, true}, {256, 512, 3, 1, 1, false, false},
                            {512, 512, 3, 1, 1, false, false}, {512, 512, 3, 1, 1, true, true},
                            {512, 512, 3, 1, 1, false, false}, {512, 512, 3, 1, 1, false, false},
                            {512, 512, 3, 1, 1, false, true}}};

constexpr int LP_LAYERS = 5;   // target layers of both networks
constexpr int BM = 128, BN = 64, BK = 32;   // conv CTA tile: 128 output pixels x 64 channels, K in steps of 32
constexpr int AS = BK + 4, BS = BN + 8;     // shared row strides: conflict-free fragment reads and float4 stores
constexpr int HEAD_PIX = 64;                // pixels per head CTA (8 warps x 8)

const LpNet* net_of(int net) { return net == GAB200_LPIPS_ALEX ? &kAlex : net == GAB200_LPIPS_VGG16 ? &kVgg : nullptr; }
int stored_channels(int cin) { return cin == 3 ? 4 : cin; }
int kpad(const LpConv& c) { return (c.ks * c.ks * stored_channels(c.cin) + BK - 1) / BK * BK; }

// Float offsets of the packed buffer: conv l's W at w[l], its bias at b[l], lin vector t at lin[t]; total floats.
struct PackPlan {
  size_t w[13], b[13], lin[LP_LAYERS], total;
};
PackPlan pack_plan(const LpNet& n) {
  PackPlan p{};
  size_t off = 0;
  int t = 0;
  for (int l = 0; l < n.nconv; l++) {
    p.w[l] = off;
    off += (size_t)kpad(n.conv[l]) * n.conv[l].cout;
    p.b[l] = off;
    off += n.conv[l].cout;
  }
  for (int l = 0; l < n.nconv; l++)
    if (n.conv[l].target) {
      p.lin[t++] = off;
      off += n.conv[l].cout;
    }
  p.total = off;
  return p;
}

// One stage of the pipeline: its output shape (per image) and where it sits among the features.
struct Stage {
  int kind;   // 0 input, 1 conv (+ bias + ReLU), 2 pool
  int conv;   // the conv index (kind 1)
  int H, W, C;
};
struct Plan {
  int nstages;
  Stage st[32];
  size_t max_floats;                  // the largest stage output of both images
  size_t head_ctas[LP_LAYERS], head_off[LP_LAYERS], partials;
  bool ok;                            // every stage has at least one output pixel
};
Plan plan_of(const LpNet& n, int H, int W) {
  Plan p{};
  p.ok = true;
  auto push = [&](int kind, int conv, int h, int w, int c) {
    if (h < 1 || w < 1) p.ok = false;
    p.st[p.nstages++] = Stage{kind, conv, h, w, c};
    const size_t f = 2 * (size_t)(h > 0 ? h : 0) * (w > 0 ? w : 0) * c;
    if (f > p.max_floats) p.max_floats = f;
  };
  push(0, -1, H, W, 4);
  int t = 0;
  for (int l = 0; l < n.nconv; l++) {
    const LpConv& c = n.conv[l];
    // floor division of a negative numerator must still mean "no output": test before dividing
    H = H + 2 * c.pad >= c.ks ? (H + 2 * c.pad - c.ks) / c.stride + 1 : 0;
    W = W + 2 * c.pad >= c.ks ? (W + 2 * c.pad - c.ks) / c.stride + 1 : 0;
    push(1, l, H, W, c.cout);
    if (c.target) {
      p.head_ctas[t] = ((size_t)(H > 0 ? H : 0) * (W > 0 ? W : 0) + HEAD_PIX - 1) / HEAD_PIX;
      p.head_off[t] = p.partials;
      p.partials += p.head_ctas[t];
      t++;
    }
    if (c.pool_after) {
      H = H >= n.pool_k ? (H - n.pool_k) / 2 + 1 : 0;
      W = W >= n.pool_k ? (W - n.pool_k) / 2 + 1 : 0;
      push(2, l, H, W, c.cout);
    }
  }
  return p;
}

__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// torch.relu: NaN stays NaN
__device__ __forceinline__ float relu(float v) { return v > 0.f ? v : (v == v ? 0.f : v); }
// max that keeps a NaN, as max_pool2d does
__device__ __forceinline__ float nanmax(float m, float v) { return (v > m || v != v) ? v : m; }

}  // namespace

// ---- weight packing ------------------------------------------------------------------------------------------------
// torchvision OIHW [Cout][Cin][ks][ks] -> [Kpad][Cout], TF32-rounded, zero where the gather reads padding.
__global__ void __launch_bounds__(256) lpips_pack_kernel(const float* __restrict__ w, int cin, int cs, int cout,
                                                          int ks, int kp, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= (int64_t)kp * cout) return;
  const int k = (int)(i / cout), n = (int)(i - (int64_t)k * cout);
  const int tap = k / cs, ci = k - tap * cs;
  float v = 0.f;
  if (tap < ks * ks && ci < cin) {
    const int ky = tap / ks, kx = tap - ky * ks;
    v = __uint_as_float(tf32_rna(w[(((int64_t)n * cin + ci) * ks + ky) * ks + kx]));
  }
  out[i] = v;
}

// ---- input ---------------------------------------------------------------------------------------------------------
// Image 0 is the render (SRC: float [3,H,W] clamped to [0, 1] as image_metrics clamps it, or the display image
// uint8 [H,W,3] read as value/255), image 1 the ground truth uint8 [3,H,W] (value/255, correctly rounded).  Each is
// z-scored as lpipsPyTorch's BaseNet.z_score: (x - mean) / std in float32.
template <int SRC>
__global__ void __launch_bounds__(256) lpips_input_kernel(int H, int W, const void* __restrict__ render,
                                                           const uint8_t* __restrict__ gt, float4* __restrict__ out) {
  __shared__ GtFetch<uint8_t> fetch;
  fetch.init(threadIdx.x);
  const int64_t hw = (int64_t)H * W;
  const int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (p >= 2 * hw) return;
  const float mean[3] = {(float)-.030, (float)-.088, (float)-.188};
  const float stdv[3] = {(float).458, (float).448, (float).450};
  float z[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float x;
    if (p >= hw) {
      x = fetch(gt, c * hw + (p - hw));
    } else if constexpr (SRC == GAB200_METRICS_FLOAT_CHW) {
      const float v = static_cast<const float*>(render)[c * hw + p];
      x = v != v ? v : fminf(fmaxf(v, 0.f), 1.f);   // torch.clamp(v, 0, 1): NaN stays NaN
    } else {
      x = fetch.tab[static_cast<const uint8_t*>(render)[p * 3 + c]];
    }
    z[c] = __fdiv_rn(__fsub_rn(x, mean[c]), stdv[c]);
  }
  out[p] = make_float4(z[0], z[1], z[2], 0.f);
}

// ---- convolution + bias + ReLU -------------------------------------------------------------------------------------
// in: NHWC [2][H][W][C] (C % 4 == 0), w: packed [Kpad][Cout] (TF32 values), out: NHWC [2][Ho][Wo][Cout].
// 8 warps as 4 (M) x 2 (N), each 32 x 32 of the 128 x 64 tile: 2 x 4 mma tiles.  The next K step's operands are
// loaded into registers while the tensor cores work on the current one in shared memory.
template <int KS, int S, int P>
__global__ void __launch_bounds__(256, 2) lpips_conv_kernel(const float* __restrict__ in, int H, int W, int C, int Ho,
                                                             int Wo, int M, int kp, int cout, int ntn,
                                                             const float* __restrict__ w,
                                                             const float* __restrict__ bias, float* __restrict__ out) {
  __shared__ __align__(16) float As[BM][AS];
  __shared__ __align__(16) float Bs[BK][BS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nt = blockIdx.x % ntn, mt = blockIdx.x / ntn;
  const int m0 = mt * BM, n0 = nt * BN;

  // A gather: this thread loads rows ar + 32 i, k offset 4 q of every K step
  const int q = tid & 7, ar = tid >> 3;
  const int hwo = Ho * Wo;
  int64_t base[4];
  int iy0[4], ix0[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int m = m0 + ar + 32 * i;
    if (m < M) {
      const int img = m / hwo, r = m - img * hwo, oy = r / Wo, ox = r - oy * Wo;
      base[i] = (int64_t)img * H * W;
      iy0[i] = oy * S - P;
      ix0[i] = ox * S - P;
    } else {   // past the last pixel: every tap reads as padding
      base[i] = 0;
      iy0[i] = -(1 << 29);
      ix0[i] = 0;
    }
  }
  // B: rows br + 16 j, columns 4 bc
  const int bc = tid & 15, br = tid >> 4;

  float4 ra[4], rb[2];
  auto load = [&](int kc) {
    const int k = kc * BK + 4 * q;
    const int tap = k / C, ci = k - tap * C;
    const int ky = tap / KS, kx = tap - ky * KS;
    const bool tap_ok = tap < KS * KS;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int iy = iy0[i] + ky, ix = ix0[i] + kx;
      ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tap_ok && (unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W)
        ra[i] = __ldg(reinterpret_cast<const float4*>(in + (base[i] + (int64_t)iy * W + ix) * C + ci));
    }
#pragma unroll
    for (int j = 0; j < 2; j++)
      rb[j] = __ldg(reinterpret_cast<const float4*>(w + (size_t)(kc * BK + br + 16 * j) * cout + n0 + 4 * bc));
  };
  auto stash = [&]() {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      float4 v;
      v.x = __uint_as_float(tf32_rna(ra[i].x));
      v.y = __uint_as_float(tf32_rna(ra[i].y));
      v.z = __uint_as_float(tf32_rna(ra[i].z));
      v.w = __uint_as_float(tf32_rna(ra[i].w));
      *reinterpret_cast<float4*>(&As[ar + 32 * i][4 * q]) = v;
    }
#pragma unroll
    for (int j = 0; j < 2; j++) *reinterpret_cast<float4*>(&Bs[br + 16 * j][4 * bc]) = rb[j];
  };

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[i][j][e] = 0.f;

  const int g = lane >> 2, t = lane & 3, wm = warp & 3, wn = warp >> 2;
  const int nk = kp / BK;
  load(0);
  stash();
  __syncthreads();
  for (int kc = 0; kc < nk; kc++) {
    if (kc + 1 < nk) load(kc + 1);
#pragma unroll
    for (int kk = 0; kk < BK; kk += 8) {
      uint32_t a[2][4], b[4][2];
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const int r = wm * 32 + i * 16 + g;
        a[i][0] = __float_as_uint(As[r][kk + t]);
        a[i][1] = __float_as_uint(As[r + 8][kk + t]);
        a[i][2] = __float_as_uint(As[r][kk + t + 4]);
        a[i][3] = __float_as_uint(As[r + 8][kk + t + 4]);
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int n = wn * 32 + j * 8 + g;
        b[j][0] = __float_as_uint(Bs[kk + t][n]);
        b[j][1] = __float_as_uint(Bs[kk + t + 4][n]);
      }
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
          asm volatile(
              "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
              "{%0,%1,%2,%3};"
              : "+f"(acc[i][j][0]), "+f"(acc[i][j][1]), "+f"(acc[i][j][2]), "+f"(acc[i][j][3])
              : "r"(a[i][0]), "r"(a[i][1]), "r"(a[i][2]), "r"(a[i][3]), "r"(b[j][0]), "r"(b[j][1]));
    }
    __syncthreads();
    if (kc + 1 < nk) {
      stash();
      __syncthreads();
    }
  }

  // epilogue: + bias (FP32), ReLU, NHWC store
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int n = n0 + wn * 32 + j * 8 + 2 * t;
    const float b0 = bias[n], b1 = bias[n + 1];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int m = m0 + wm * 32 + i * 16 + g + 8 * h;
        if (m < M)
          *reinterpret_cast<float2*>(out + (size_t)m * cout + n) =
              make_float2(relu(acc[i][j][2 * h] + b0), relu(acc[i][j][2 * h + 1] + b1));
      }
  }
}

// ---- max pool ------------------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(256) lpips_pool_kernel(const float4* __restrict__ in, int H, int W, int c4, int Ho,
                                                          int Wo, float4* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int64_t total = 2 * (int64_t)Ho * Wo * c4;
  if (i >= total) return;
  const int c = (int)(i % c4);
  const int64_t p = i / c4;
  const int64_t hwo = (int64_t)Ho * Wo;
  const int img = (int)(p / hwo);
  const int r = (int)(p - img * hwo), oy = r / Wo, ox = r - oy * Wo;
  const float4* src = in + (((int64_t)img * H + 2 * oy) * W + 2 * ox) * c4 + c;
  float4 m = src[0];
#pragma unroll
  for (int ky = 0; ky < K; ky++)
#pragma unroll
    for (int kx = 0; kx < K; kx++) {
      const float4 v = src[((int64_t)ky * W + kx) * c4];
      m.x = nanmax(m.x, v.x);
      m.y = nanmax(m.y, v.y);
      m.z = nanmax(m.z, v.z);
      m.w = nanmax(m.w, v.w);
    }
  out[i] = m;
}

// ---- head ----------------------------------------------------------------------------------------------------------
// feat: NHWC [2][hw][C] post-ReLU features.  One warp per pixel: f / (sqrt(sum f^2) + 1e-10) of both images, the
// squared difference, the lin dot product -- FP32, as lpipsPyTorch's normalize_activation and LinLayers.
__global__ void __launch_bounds__(256) lpips_head_kernel(const float* __restrict__ feat, int64_t hw, int C,
                                                          const float* __restrict__ lin,
                                                          double* __restrict__ partial) {
  __shared__ double part[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc = 0.0;
  for (int k = 0; k < HEAD_PIX / 8; k++) {
    const int64_t p = (int64_t)blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + k;
    if (p >= hw) break;
    const float* fx = feat + p * C;
    const float* fy = feat + (hw + p) * C;
    float sx = 0.f, sy = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float x = fx[c], y = fy[c];
      sx += x * x;
      sy += y * y;
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
      sx += __shfl_xor_sync(0xffffffffu, sx, m);
      sy += __shfl_xor_sync(0xffffffffu, sy, m);
    }
    const float dx = sqrtf(sx) + 1e-10f, dy = sqrtf(sy) + 1e-10f;
    float v = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float d = fx[c] / dx - fy[c] / dy;
      v += lin[c] * (d * d);
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    acc += (double)v;
  }
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < 8; w++) s += part[w];
    partial[blockIdx.x] = s;
  }
}

struct HeadSums {
  int64_t count[LP_LAYERS], offset[LP_LAYERS];
  double inv_n[LP_LAYERS];
};

__global__ void __launch_bounds__(256) lpips_finalize_kernel(HeadSums h, const double* __restrict__ partial,
                                                              const int32_t* __restrict__ row, int rows,
                                                              const int32_t* __restrict__ skip,
                                                              float* __restrict__ table) {
  if (skip != nullptr && *skip != 0) return;   // uniform over the CTA
  const int r = row != nullptr ? *row : 0;
  if (r < 0 || r >= rows) return;
  __shared__ double part[LP_LAYERS][8];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  double v[LP_LAYERS];
#pragma unroll
  for (int l = 0; l < LP_LAYERS; l++) {
    double s = 0.0;
    for (int64_t i = tid; i < h.count[l]; i += 256) s += partial[h.offset[l] + i];
    v[l] = s;
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1)
#pragma unroll
    for (int l = 0; l < LP_LAYERS; l++) v[l] += __shfl_xor_sync(0xffffffffu, v[l], m);
  if (lane == 0)
#pragma unroll
    for (int l = 0; l < LP_LAYERS; l++) part[l][wrp] = v[l];
  __syncthreads();
  if (tid == 0) {
    double total = 0.0;
#pragma unroll
    for (int l = 0; l < LP_LAYERS; l++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++) s += part[l][w];
      total += s * h.inv_n[l];
    }
    table[r] = (float)total;
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------
static unsigned blocks(int64_t n) { return (unsigned)((n + 255) / 256); }

size_t lpips_weights_bytes(int net) {
  const LpNet* n = net_of(net);
  return n ? pack_plan(*n).total * sizeof(float) : 0;
}

size_t lpips_scratch_bytes(int net, int H, int W) {
  const LpNet* n = net_of(net);
  if (!n || H < 1 || W < 1) return 0;
  const Plan p = plan_of(*n, H, W);
  if (!p.ok) return 0;
  // the partials first (8-byte), then two activation buffers, each 16-byte aligned
  const size_t head = (p.partials * sizeof(double) + 15) / 16 * 16;
  return head + 2 * p.max_floats * sizeof(float);
}

size_t lpips_features_bytes(int net, int H, int W) {
  const LpNet* n = net_of(net);
  if (!n || H < 1 || W < 1) return 0;
  const Plan p = plan_of(*n, H, W);
  if (!p.ok) return 0;
  size_t f = 0;
  for (int s = 0; s < p.nstages; s++) f += 2 * (size_t)p.st[s].H * p.st[s].W * p.st[s].C;
  return f * sizeof(float);
}

int lpips_conv_count(int net) {
  const LpNet* n = net_of(net);
  return n ? n->nconv : 0;
}

void launch_lpips_pack(int net, const float* const* conv_w, const float* const* conv_b, const float* const* lin,
                       float* packed, cudaStream_t stream) {
  const LpNet& n = *net_of(net);
  const PackPlan pp = pack_plan(n);
  int t = 0;
  for (int l = 0; l < n.nconv; l++) {
    const LpConv& c = n.conv[l];
    const int kp = kpad(c);
    lpips_pack_kernel<<<blocks((int64_t)kp * c.cout), 256, 0, stream>>>(conv_w[l], c.cin, stored_channels(c.cin),
                                                                         c.cout, c.ks, kp, packed + pp.w[l]);
    count_launch();
    cudaMemcpyAsync(packed + pp.b[l], conv_b[l], c.cout * sizeof(float), cudaMemcpyDeviceToDevice, stream);
    if (c.target) {
      cudaMemcpyAsync(packed + pp.lin[t], lin[t], c.cout * sizeof(float), cudaMemcpyDeviceToDevice, stream);
      t++;
    }
  }
}

static void launch_conv(const LpConv& c, const float* in, int H, int W, int C, int Ho, int Wo, const float* w,
                        const float* b, float* out, cudaStream_t stream) {
  const int M = 2 * Ho * Wo, ntn = c.cout / BN;
  const unsigned grid = (unsigned)(((int64_t)M + BM - 1) / BM * ntn);
  const int kp = kpad(c);
  if (c.ks == 11)
    lpips_conv_kernel<11, 4, 2><<<grid, 256, 0, stream>>>(in, H, W, C, Ho, Wo, M, kp, c.cout, ntn, w, b, out);
  else if (c.ks == 5)
    lpips_conv_kernel<5, 1, 2><<<grid, 256, 0, stream>>>(in, H, W, C, Ho, Wo, M, kp, c.cout, ntn, w, b, out);
  else
    lpips_conv_kernel<3, 1, 1><<<grid, 256, 0, stream>>>(in, H, W, C, Ho, Wo, M, kp, c.cout, ntn, w, b, out);
  count_launch();
}

void launch_lpips(const gab200_lpips_args& a, cudaStream_t stream) {
  const LpNet& n = *net_of(a.net);
  const PackPlan pp = pack_plan(n);
  const Plan p = plan_of(n, a.height, a.width);
  const float* wts = static_cast<const float*>(a.weights);
  double* partial = static_cast<double*>(a.scratch);
  float* buf[2];
  buf[0] = reinterpret_cast<float*>(static_cast<char*>(a.scratch) + (p.partials * sizeof(double) + 15) / 16 * 16);
  buf[1] = buf[0] + p.max_floats;
  // with a.features every stage writes its own slice of it; else the stages alternate between the two buffers
  float* feat = a.features;
  auto dst = [&](int s) -> float* {
    if (feat == nullptr) return buf[s & 1];
    float* d = feat;
    feat += 2 * (size_t)p.st[s].H * p.st[s].W * p.st[s].C;
    return d;
  };

  float* cur = dst(0);
  const int64_t px = 2 * (int64_t)a.height * a.width;
  if (a.render_kind == GAB200_METRICS_FLOAT_CHW)
    lpips_input_kernel<GAB200_METRICS_FLOAT_CHW><<<blocks(px), 256, 0, stream>>>(
        a.height, a.width, a.render, a.gt, reinterpret_cast<float4*>(cur));
  else
    lpips_input_kernel<GAB200_METRICS_U8_HWC><<<blocks(px), 256, 0, stream>>>(
        a.height, a.width, a.render, a.gt, reinterpret_cast<float4*>(cur));
  count_launch();

  HeadSums h{};
  int t = 0;
  for (int s = 1; s < p.nstages; s++) {
    const Stage& in = p.st[s - 1];
    const Stage& st = p.st[s];
    float* out = dst(s);
    if (st.kind == 1) {
      const LpConv& c = n.conv[st.conv];
      launch_conv(c, cur, in.H, in.W, in.C, st.H, st.W, wts + pp.w[st.conv], wts + pp.b[st.conv], out, stream);
      if (c.target) {
        lpips_head_kernel<<<(unsigned)p.head_ctas[t], 256, 0, stream>>>(out, (int64_t)st.H * st.W, st.C,
                                                                        wts + pp.lin[t], partial + p.head_off[t]);
        count_launch();
        h.count[t] = (int64_t)p.head_ctas[t];
        h.offset[t] = (int64_t)p.head_off[t];
        h.inv_n[t] = 1.0 / ((double)st.H * st.W);   // the mean multiplies by a reciprocal formed here
        t++;
      }
    } else {
      const int c4 = st.C / 4;
      const unsigned g = blocks(2 * (int64_t)st.H * st.W * c4);
      if (n.pool_k == 3)
        lpips_pool_kernel<3><<<g, 256, 0, stream>>>(reinterpret_cast<const float4*>(cur), in.H, in.W, c4, st.H, st.W,
                                                    reinterpret_cast<float4*>(out));
      else
        lpips_pool_kernel<2><<<g, 256, 0, stream>>>(reinterpret_cast<const float4*>(cur), in.H, in.W, c4, st.H, st.W,
                                                    reinterpret_cast<float4*>(out));
      count_launch();
    }
    cur = out;
  }
  lpips_finalize_kernel<<<1, 256, 0, stream>>>(h, partial, a.row, a.table_rows, a.skip_flag, a.table);
  count_launch();
}

}  // namespace gab
