// optim.cu -- Adam on the splat arrays as ONE multi-tensor launch (SURVEY.md 8f rank 3).
//
// The reference steps `torch.optim.Adam(l, lr=0.0, eps=1e-15)` over six parameter groups with per-group learning rates
// (scene/gaussian_model.py:213-232, train.py:207-209): ~10 eager kernels per group per step in the default
// implementation.  The update is pure HBM streaming -- read p, g, m, v (16 B), write p, m, v (12 B) per element --
// so all groups go through one grid-stride kernel with 128-bit accesses; `blockIdx.y` picks the group.
//
// Arithmetic follows torch's single-tensor Adam (torch/optim/adam.py, amsgrad=False, weight_decay=0, maximize=False):
//   m <- m + (g - m) (1 - beta1)                 (Tensor.lerp_)
//   v <- beta2 v + (1 - beta2) g g               (mul_ / addcmul_)
//   p <- p - (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
// The scalars (1 - beta, lr / (1 - beta1^t), ...) are formed on the host in double from double hyper-parameters, as
// torch forms them from Python floats, and rounded to float once: 1.0f - 0.999f would already be off by 1.3e-5.
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

struct AdamBatch {
  float* p[GAB_ADAM_MAX_SEGMENTS];
  const float* g[GAB_ADAM_MAX_SEGMENTS];
  float* m[GAB_ADAM_MAX_SEGMENTS];
  float* v[GAB_ADAM_MAX_SEGMENTS];
  int64_t n[GAB_ADAM_MAX_SEGMENTS];
  float step_size[GAB_ADAM_MAX_SEGMENTS];  // lr / bias_correction1
  int32_t vec4[GAB_ADAM_MAX_SEGMENTS];     // bit 0: p, m, v 16-byte aligned (128-bit path); bit 1: g aligned too
};

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float w1, float beta2, float w2,
                                         float inv_bc2_sqrt, float eps, float step_size) {
  m = m + (g - m) * w1;
  v = v * beta2 + (w2 * g) * g;
  const float denom = sqrtf(v) * inv_bc2_sqrt + eps;
  p = p - step_size * (m / denom);
}

// One segment's grid-stride update: the body of both launches below.
__device__ __forceinline__ void adam_segment(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                             float* __restrict__ v, int64_t n, int32_t vec4, float w1, float beta2,
                                             float w2, float inv_bc2_sqrt, float eps, float step_size) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t tail = 0;
  if (vec4 & 1) {
    // the gradient is usually a view into the fused backward's flat buffer: its offset need not be 16-byte aligned
    const bool g_vec = (vec4 & 2) != 0;
    const int64_t n4 = n >> 2;
    auto load_g = [&](int64_t i) {
      return g_vec ? reinterpret_cast<const float4*>(g)[i] : make_float4(g[4 * i], g[4 * i + 1], g[4 * i + 2], g[4 * i + 3]);
    };
    auto update = [&](float4& P, const float4& G, float4& M, float4& V) {
      adam_one(P.x, G.x, M.x, V.x, w1, beta2, w2, inv_bc2_sqrt, eps, step_size);
      adam_one(P.y, G.y, M.y, V.y, w1, beta2, w2, inv_bc2_sqrt, eps, step_size);
      adam_one(P.z, G.z, M.z, V.z, w1, beta2, w2, inv_bc2_sqrt, eps, step_size);
      adam_one(P.w, G.w, M.w, V.w, w1, beta2, w2, inv_bc2_sqrt, eps, step_size);
    };
    int64_t i = t0;
    for (; i + stride < n4; i += 2 * stride) {  // two independent 4 x 16 B load groups in flight per thread
      const int64_t j = i + stride;
      float4 P0 = reinterpret_cast<float4*>(p)[i], P1 = reinterpret_cast<float4*>(p)[j];
      const float4 G0 = load_g(i), G1 = load_g(j);
      float4 M0 = reinterpret_cast<float4*>(m)[i], M1 = reinterpret_cast<float4*>(m)[j];
      float4 V0 = reinterpret_cast<float4*>(v)[i], V1 = reinterpret_cast<float4*>(v)[j];
      update(P0, G0, M0, V0);
      update(P1, G1, M1, V1);
      reinterpret_cast<float4*>(p)[i] = P0; reinterpret_cast<float4*>(p)[j] = P1;
      reinterpret_cast<float4*>(m)[i] = M0; reinterpret_cast<float4*>(m)[j] = M1;
      reinterpret_cast<float4*>(v)[i] = V0; reinterpret_cast<float4*>(v)[j] = V1;
    }
    if (i < n4) {
      float4 P = reinterpret_cast<float4*>(p)[i];
      const float4 G = load_g(i);
      float4 M = reinterpret_cast<float4*>(m)[i];
      float4 V = reinterpret_cast<float4*>(v)[i];
      update(P, G, M, V);
      reinterpret_cast<float4*>(p)[i] = P;
      reinterpret_cast<float4*>(m)[i] = M;
      reinterpret_cast<float4*>(v)[i] = V;
    }
    tail = n4 << 2;
  }
  for (int64_t i = tail + t0; i < n; i += stride) {
    float P = p[i], M = m[i], V = v[i];
    adam_one(P, g[i], M, V, w1, beta2, w2, inv_bc2_sqrt, eps, step_size);
    p[i] = P;
    m[i] = M;
    v[i] = V;
  }
}

__global__ void __launch_bounds__(256) adam_kernel(AdamBatch b, float w1, float beta2, float w2, float inv_bc2_sqrt,
                                                   float eps) {
  const int s = blockIdx.y;
  adam_segment(b.p[s], b.g[s], b.m[s], b.v[s], b.n[s], b.vec4[s], w1, beta2, w2, inv_bc2_sqrt, eps, b.step_size[s]);
}

void launch_adam(int num_segments, const gab200_adam_segment* segs, int64_t step, double beta1, double beta2, double eps,
                 cudaStream_t stream) {
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  const float inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
  int next = 0;  // first input segment not yet consumed (empty segments are skipped without filling a slot)
  while (next < num_segments) {
    AdamBatch b;
    int cnt = 0;
    int64_t longest = 0;
    for (; next < num_segments && cnt < GAB_ADAM_MAX_SEGMENTS; next++) {
      const gab200_adam_segment& s = segs[next];
      if (s.n <= 0) continue;
      b.p[cnt] = s.param;
      b.g[cnt] = s.grad;
      b.m[cnt] = s.exp_avg;
      b.v[cnt] = s.exp_avg_sq;
      b.n[cnt] = s.n;
      b.step_size[cnt] = (float)(s.lr / bc1);
      const uintptr_t bits = (uintptr_t)s.param | (uintptr_t)s.exp_avg | (uintptr_t)s.exp_avg_sq;
      b.vec4[cnt] = (bits & 15) == 0 ? (((uintptr_t)s.grad & 15) == 0 ? 3 : 1) : 0;
      longest = s.n > longest ? s.n : longest;
      cnt++;
    }
    if (cnt == 0) continue;
    for (int i = cnt; i < GAB_ADAM_MAX_SEGMENTS; i++) {
      b.p[i] = nullptr; b.g[i] = nullptr; b.m[i] = nullptr; b.v[i] = nullptr;
      b.n[i] = 0; b.step_size[i] = 0.f; b.vec4[i] = 0;
    }
    // two float4 per thread for the longest group, capped at 8 waves of GAB_NUM_SMS SMs x 8 resident CTAs
    int64_t blocks = (longest / 8 + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > GAB_NUM_SMS * 8 * 8) blocks = GAB_NUM_SMS * 8 * 8;
    adam_kernel<<<dim3((unsigned)blocks, (unsigned)cnt), 256, 0, stream>>>(
        b, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), inv_bc2_sqrt, (float)eps);
    count_launch();
  }
}

// ---- capturable variant: every per-step scalar is formed on the device --------------------------------------------
struct AdamDeviceBatch {
  gab200_adam_device_segment seg[GAB_ADAM_MAX_SEGMENTS];
  int32_t vec4[GAB_ADAM_MAX_SEGMENTS];
};

__device__ __forceinline__ bool skipped(const int32_t* skip) { return skip != nullptr && *skip != 0; }

// get_expon_lr_func (utils/general_utils.py) in double, operation for operation: __dmul_rn / __dadd_rn keep the compiler
// from contracting a * b + c into one fma, which numpy does not do either.
__device__ double expon_lr(const gab200_adam_device_segment& s, double step) {
  if (step < 0.0 || (s.lr_init == 0.0 && s.lr_final == 0.0)) return 0.0;
  double delay_rate = 1.0;
  if (s.lr_delay_steps > 0) {
    const double x = fmin(fmax(step / (double)s.lr_delay_steps, 0.0), 1.0);
    delay_rate = __dadd_rn(s.lr_delay_mult, __dmul_rn(1.0 - s.lr_delay_mult, sin(__dmul_rn(0.5 * M_PI, x))));
  }
  const double t = fmin(fmax(step / (double)s.max_steps, 0.0), 1.0);
  const double log_lerp = exp(__dadd_rn(__dmul_rn(log(s.lr_init), 1.0 - t), __dmul_rn(log(s.lr_final), t)));
  return __dmul_rn(delay_rate, log_lerp);
}

// A separate single-thread launch: if the Adam kernel incremented the counter itself, its other blocks could read
// either the old or the new value.
__global__ void adam_count_step_kernel(AdamDeviceBatch b, int cnt, const int32_t* __restrict__ skip) {
  if (skipped(skip)) return;
  for (int s = 0; s < cnt; s++) *b.seg[s].step += 1.0f;
}

__global__ void __launch_bounds__(256) adam_device_kernel(AdamDeviceBatch b, double beta1, double beta2, float w1,
                                                          float beta2f, float w2, float eps,
                                                          const int32_t* __restrict__ skip) {
  if (skipped(skip)) return;
  const int s = blockIdx.y;
  const gab200_adam_device_segment& sg = b.seg[s];
  __shared__ float scal[2];  // lr / bias_correction1, 1 / sqrt(bias_correction2): launch_adam's host arithmetic
  if (threadIdx.x == 0) {
    const double step = (double)*sg.step;
    const double lr = sg.has_schedule ? expon_lr(sg, step) : sg.lr;
    const double bc1 = 1.0 - pow(beta1, step);
    const double bc2 = 1.0 - pow(beta2, step);
    scal[0] = (float)(lr / bc1);
    scal[1] = (float)(1.0 / sqrt(bc2));
  }
  __syncthreads();
  adam_segment(sg.param, sg.grad, sg.exp_avg, sg.exp_avg_sq, sg.n, b.vec4[s], w1, beta2f, w2, scal[1], eps, scal[0]);
}

void launch_adam_device(int num_segments, const gab200_adam_device_segment* segs, double beta1, double beta2,
                        double eps, const int32_t* skip, cudaStream_t stream) {
  for (int first = 0; first < num_segments; first += GAB_ADAM_MAX_SEGMENTS) {
    AdamDeviceBatch b;
    memset(&b, 0, sizeof(b));
    const int cnt = num_segments - first < GAB_ADAM_MAX_SEGMENTS ? num_segments - first : GAB_ADAM_MAX_SEGMENTS;
    int64_t longest = 0;
    for (int i = 0; i < cnt; i++) {
      const gab200_adam_device_segment& s = segs[first + i];
      b.seg[i] = s;
      const uintptr_t bits = (uintptr_t)s.param | (uintptr_t)s.exp_avg | (uintptr_t)s.exp_avg_sq;
      b.vec4[i] = (bits & 15) == 0 ? (((uintptr_t)s.grad & 15) == 0 ? 3 : 1) : 0;
      longest = s.n > longest ? s.n : longest;
    }
    adam_count_step_kernel<<<1, 1, 0, stream>>>(b, cnt, skip);
    count_launch();
    int64_t blocks = (longest / 8 + 255) / 256;  // the grid of launch_adam
    if (blocks < 1) blocks = 1;
    if (blocks > GAB_NUM_SMS * 8 * 8) blocks = GAB_NUM_SMS * 8 * 8;
    adam_device_kernel<<<dim3((unsigned)blocks, (unsigned)cnt), 256, 0, stream>>>(
        b, beta1, beta2, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, skip);
    count_launch();
  }
}

}  // namespace gab
