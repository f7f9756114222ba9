// preprocess.cu -- per-splat forward stage with the FLAME mesh binding fused in, plus tile|depth key emission
// and tile-range detection.  COMPILED WITH --fmad=false: every float expression rounds exactly as written
// (IEEE rn, no contraction), and the association of every sum is the documented left-to-right order, so the
// depth bits, pixel centres, radii and tile rectangles -- hence the tile|depth keys -- are reproducible bit for
// bit by the CPU oracle (oracle/splat_oracle.c, built with -ffp-contract=off).
//
// Replaces, in ONE kernel (SURVEY.md 2.4 K1 + the eager getters of 2.4(b)):
//   scene/gaussian_model.py:113-160   get_xyz / get_rotation / get_scaling / get_opacity / get_features
//   diff_gaussian_rasterization preprocessCUDA (absent submodule; behaviour: SURVEY.md Appendix B.1)
#include "common.cuh"
#include "kernels.cuh"
#include "splat_math.cuh"

namespace gab {

#define REC_SCALE_AC (-0.5f * 1.4426950408889634f)
#define REC_SCALE_B (-1.4426950408889634f)

// =====================================================================================================
// K1: fused bind + activate + project + EWA + SH->RGB.  One thread per splat.
// CAM (splat_math.cuh): CAM_TABLE renders row blockIdx.y of the camera table; outputs at the virtual splat
// view * P + i, tile counts in the view's slice.
// DA: the record also carries the view-space depth z in q2.w, read by the depth plane of the blend (forward and
// backward).  clamped != nullptr: the per-channel colour clamp bits, which the backward reads.
// =====================================================================================================
template <bool BOUND, int CAM, bool DA>
__global__ void __launch_bounds__(PRE_NT) preprocess_kernel(gab200_forward_args a, const float* __restrict__ cameras,
                                                            const float* __restrict__ tanfov, SplatRec* __restrict__ rec,
                                                            SplatAux* __restrict__ aux,
                                                            uint32_t* __restrict__ tiles_touched,
                                                            uint8_t* __restrict__ clamped,
                                                            uint32_t* __restrict__ depth_keys,
                                                            uint32_t* __restrict__ ids, int exact_binning,
                                                            DepthBuckets bk, uint32_t* __restrict__ tile_count) {
  __shared__ Camera cam;
  __shared__ float sh_s[PRE_NT * SH_SMEM_STRIDE_MAX];
  const int view = CAM == CAM_TABLE ? (int)blockIdx.y : 0;
  pdl_wait();
  pdl_trigger();
  if (CAM == CAM_TABLE) {
    const float* row = cameras + (size_t)view * GAB200_CAMERA_FLOATS;
    stage_camera(row, row + 16, row + 32, cam);
    tanfov = row + 35;
    const int view_tiles = ((a.image_width + GAB_TILE - 1) / GAB_TILE) * ((a.image_height + GAB_TILE - 1) / GAB_TILE);
    if (tile_count != nullptr) tile_count += view * view_tiles;
  } else {
    stage_camera(a.viewmatrix, a.projmatrix, a.campos, cam);
  }
  // SH coefficients of the block's splats: coalesced 128-bit loads -> shared memory (row stride odd: conflict-free)
  const int sh_width = BOUND ? 3 * (a.sh_coeffs - 1) : 3 * a.sh_coeffs;
  const int sh_stride = sh_width | 1;
  const float* sh_src = BOUND ? a.sh_rest : a.shs;
  const bool use_sh = a.colors_precomp == nullptr && sh_src != nullptr && sh_width > 0;
  if (use_sh) {
    const int row0 = blockIdx.x * PRE_NT;
    stage_rows_in<PRE_NT>(sh_s, sh_src, (size_t)row0, min(PRE_NT, a.P - row0), sh_width, sh_stride);
    __syncthreads();
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  const int o = CAM == CAM_TABLE ? view * a.P + i : i;  // where the outputs of splat i go; inputs are read at i
  // the other 44 bytes per splat: quaternion as one LDG.128, positions / scales / opacity as coalesced scalar loads
  // (staging them would cost a barrier for 24 of the 284 bytes)
  RawAttr raw;
  load_raw(a, i, raw);
  const float* my_sh = sh_s + threadIdx.x * sh_stride;
  const int W = a.image_width, H = a.image_height;
  const int gx = (W + GAB_TILE - 1) / GAB_TILE, gy = (H + GAB_TILE - 1) / GAB_TILE;

  SplatRec out;
  out.q0 = make_float4(0.f, 0.f, 0.f, 0.f);
  out.q1 = make_float4(0.f, 0.f, 0.f, 0.f);
  out.q2 = make_float4(0.f, 0.f, 0.f, 0.f);
  int radius_out = 0;
  float depth_out = 0.f;
  uint32_t tiles_out = 0;
  uint8_t clamp_bits = 0;

  float3 p;
  float opacity;
  float c3[6];
  bool have_cov = false;
  if (BOUND) {
    Activated act;
    BindCtx bctx;
    bind_activate(a, i, raw, act, bctx);
    p = act.mean;
    opacity = act.opacity;
    float s[3] = {a.scale_modifier * act.s[0], a.scale_modifier * act.s[1], a.scale_modifier * act.s[2]};
    cov3d_from_R(act.R, s, c3);
    have_cov = true;
  } else {
    p = make_float3(raw.x[0], raw.x[1], raw.x[2]);
    opacity = raw.o;
  }

  // a device field of view: one broadcast load per thread; a device value that is zero, negative or not finite culls the splat
  // before any tile index is formed (radius 0, no instances)
  float dev_tx = 0.f, dev_ty = 0.f;
  bool fov_ok = true;
  if (CAM != CAM_ARGS) {
    dev_tx = __ldg(tanfov);
    dev_ty = __ldg(tanfov + 1);
    fov_ok = dev_tx > 0.f && isfinite(dev_tx) && dev_ty > 0.f && isfinite(dev_ty);
  }
  const float3 t = xform4x3(cam.V, p);
  if (fov_ok && t.z > 0.2f) {
    const float hx = cam.Pm[0] * p.x + cam.Pm[4] * p.y + cam.Pm[8] * p.z + cam.Pm[12];
    const float hy = cam.Pm[1] * p.x + cam.Pm[5] * p.y + cam.Pm[9] * p.z + cam.Pm[13];
    const float hw = cam.Pm[3] * p.x + cam.Pm[7] * p.y + cam.Pm[11] * p.z + cam.Pm[15];
    const float p_w = 1.0f / (hw + 0.0000001f);
    const float ndc_x = hx * p_w, ndc_y = hy * p_w;

    if (!have_cov) {
      if (a.cov3D_precomp != nullptr) {
#pragma unroll
        for (int k = 0; k < 6; k++) c3[k] = a.cov3D_precomp[6 * (size_t)i + k];
      } else {
        float R[9];
        quat_to_R(raw.q[0], raw.q[1], raw.q[2], raw.q[3], R);
        float s[3] = {a.scale_modifier * raw.s[0], a.scale_modifier * raw.s[1], a.scale_modifier * raw.s[2]};
        cov3d_from_R(R, s, c3);
      }
    }

    const float tanfovx = CAM != CAM_ARGS ? dev_tx : a.tanfovx, tanfovy = CAM != CAM_ARGS ? dev_ty : a.tanfovy;
    const float focal_x = (float)W / (2.0f * tanfovx), focal_y = (float)H / (2.0f * tanfovy);
    const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
    const float txtz = t.x / t.z, tytz = t.y / t.z;
    const float tcx = fminf(limx, fmaxf(-limx, txtz)) * t.z;
    const float tcy = fminf(limy, fmaxf(-limy, tytz)) * t.z;
    const float j00 = focal_x / t.z, j02 = -(focal_x * tcx) / (t.z * t.z);
    const float j11 = focal_y / t.z, j12 = -(focal_y * tcy) / (t.z * t.z);
    float T0[3], T1[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      T0[c] = j00 * cam.V[4 * c + 0] + j02 * cam.V[4 * c + 2];
      T1[c] = j11 * cam.V[4 * c + 1] + j12 * cam.V[4 * c + 2];
    }
    const float S[9] = {c3[0], c3[1], c3[2], c3[1], c3[3], c3[4], c3[2], c3[4], c3[5]};
    float u[3], v[3];
#pragma unroll
    for (int r = 0; r < 3; r++) {
      u[r] = S[3 * r + 0] * T0[0] + S[3 * r + 1] * T0[1] + S[3 * r + 2] * T0[2];
      v[r] = S[3 * r + 0] * T1[0] + S[3 * r + 1] * T1[1] + S[3 * r + 2] * T1[2];
    }
    float ca = T0[0] * u[0] + T0[1] * u[1] + T0[2] * u[2];
    float cb = T0[0] * v[0] + T0[1] * v[1] + T0[2] * v[2];
    float cc = T1[0] * v[0] + T1[1] * v[1] + T1[2] * v[2];
    ca += 0.3f;
    cc += 0.3f;
    const float det = ca * cc - cb * cb;
    if (det != 0.0f) {
      const float det_inv = 1.f / det;
      const float conic_x = cc * det_inv, conic_y = -cb * det_inv, conic_z = ca * det_inv;
      const float mid = 0.5f * (ca + cc);
      const float sq = sqrtf(fmaxf(0.1f, mid * mid - det));
      const float lambda1 = mid + sq, lambda2 = mid - sq;
      const float my_radius = ceilf(3.f * sqrtf(fmaxf(lambda1, lambda2)));
      const float px = ndc2pix(ndc_x, W), py = ndc2pix(ndc_y, H);
      int x0, y0, x1, y1;
      tile_rect(px, py, (int)my_radius, gx, gy, x0, y0, x1, y1);
      if ((x1 - x0) * (y1 - y0) != 0) {
        float rgb[3];
        if (a.colors_precomp != nullptr) {
          rgb[0] = a.colors_precomp[3 * (size_t)i];
          rgb[1] = a.colors_precomp[3 * (size_t)i + 1];
          rgb[2] = a.colors_precomp[3 * (size_t)i + 2];
        } else {
          float3 d = make_float3(p.x - cam.campos[0], p.y - cam.campos[1], p.z - cam.campos[2]);
          const float len = sqrtf(d.x * d.x + d.y * d.y + d.z * d.z);
          d.x = d.x / len; d.y = d.y / len; d.z = d.z / len;
          float B[16];
          sh_basis(a.sh_degree, d, B);
          const int nb = (a.sh_degree + 1) * (a.sh_degree + 1);
          float acc[3] = {0.f, 0.f, 0.f};
          if (BOUND) {
            const float* dc = a.sh_dc + 3 * (size_t)i;
            acc[0] = acc[0] + B[0] * dc[0];
            acc[1] = acc[1] + B[0] * dc[1];
            acc[2] = acc[2] + B[0] * dc[2];
            const float* rest = my_sh;
            for (int k = 1; k < nb; k++) {
              acc[0] = acc[0] + B[k] * rest[3 * (k - 1) + 0];
              acc[1] = acc[1] + B[k] * rest[3 * (k - 1) + 1];
              acc[2] = acc[2] + B[k] * rest[3 * (k - 1) + 2];
            }
          } else {
            const float* sh = my_sh;
            for (int k = 0; k < nb; k++) {
              acc[0] = acc[0] + B[k] * sh[3 * k + 0];
              acc[1] = acc[1] + B[k] * sh[3 * k + 1];
              acc[2] = acc[2] + B[k] * sh[3 * k + 2];
            }
          }
#pragma unroll
          for (int ch = 0; ch < 3; ch++) {
            float r = acc[ch] + 0.5f;
            if (r < 0.f) clamp_bits |= (1u << ch);
            rgb[ch] = fmaxf(r, 0.f);
          }
        }
        radius_out = (int)my_radius;
        // conic pre-scaled for the blend kernels' exponent in log2 units: pw = A' dx^2 + B' dx dy + C' dy^2
        out.q0 = make_float4(px, py, conic_x * REC_SCALE_AC, conic_y * REC_SCALE_B);
        out.q1 = make_float4(conic_z * REC_SCALE_AC, opacity, rgb[0], rgb[1]);
        // the span test must see exactly the values key emission will read back from the record
        TileSpan span(px, py, (conic_x * REC_SCALE_AC) / REC_SCALE_AC, (conic_y * REC_SCALE_B) / REC_SCALE_B,
                      (conic_z * REC_SCALE_AC) / REC_SCALE_AC, opacity, x0, x1);
        const float ext_x = !span.any ? -1.f : (span.full ? 1.0e30f : span.dxmax + 0.02f);
        const float ext_y = !span.any ? -1.f : (span.full ? 1.0e30f : span.ymax + 0.02f);
        // instance count of the splat; with `tile_count` (counting tile sort, tile_sort.cu) also one RED per instance
        // into its tile's counter, so that the tile ranges exist before anything is emitted
        if (exact_binning) {
          tiles_out = (uint32_t)((y1 - y0) * (x1 - x0));
          if (tile_count != nullptr)
            for (int ty = y0; ty < y1; ty++)
              for (int x = x0; x < x1; x++) atomicAdd(tile_count + ty * gx + x, 1u);
        } else {
          uint32_t cnt = 0;
          if (span.any)
            for (int ty = y0; ty < y1; ty++) {
              int cx0, cx1;
              span.row(ty, cx0, cx1);
              cnt += (uint32_t)(cx1 - cx0);
              if (tile_count != nullptr)
                for (int x = cx0; x < cx1; x++) atomicAdd(tile_count + ty * gx + x, 1u);
            }
          tiles_out = cnt;
        }
        // DA: z for the depth plane, the float the depth key is made from
        out.q2 = make_float4(rgb[2], ext_x, ext_y, DA ? t.z : 0.f);
        depth_out = t.z;
      }
    }
  }
  // stage-A sort input: the fp32 depth bit pattern (splats that emit nothing go last), value = splat id
  const uint32_t dkey = tiles_out ? __float_as_uint(depth_out) : 0xffffffffu;
  depth_keys[o] = dkey;
  ids[o] = (uint32_t)o;
  {
    // key range of this frame (the caller's hint for the next one) and, with a hint, the bucket histogram + the
    // splat's arrival rank in its bucket (binning.cu header)
    const unsigned live = __activemask();
    const uint32_t kmin = __reduce_min_sync(live, dkey);
    const uint32_t kmax = __reduce_max_sync(live, tiles_out ? dkey : 0u);
    const uint32_t warp_tiles = __reduce_add_sync(live, tiles_out);  // <= 32 x (tiles of the image): fits 32 bits
    if ((threadIdx.x & 31) == (__ffs(live) - 1) && kmin != 0xffffffffu) {
      atomicMax(bk.meta + 0, ~kmin);
      atomicMax(bk.meta + 1, kmax);
      // 64-bit instance total: the 32-bit emission offsets / tile ranges wrap silently beyond 2^32 - 1 instances,
      // the host turns a non-zero high word into GAB200_ERR_OVERFLOW
      atomicAdd(reinterpret_cast<unsigned long long*>(bk.meta + GAB_META_TOTAL64), (unsigned long long)warp_tiles);
    }
    if (bk.enabled && tiles_out) {
      const uint32_t b = depth_bucket(dkey, bk);
      bk.rank[o] = atomicAdd(bk.counts + b, 1u);
      atomicAdd(bk.tiles + b, tiles_out);
    }
  }
  rec[o] = out;
  SplatAux ax;
  ax.depth = depth_out; ax.radius = radius_out; ax.tiles = tiles_out; ax.pad = 0;
  aux[o] = ax;
  a.radii[o] = radius_out;
  if (a.visibility != nullptr) a.visibility[o] = radius_out > 0 ? 1 : 0;
  tiles_touched[o] = tiles_out;
  if (clamped != nullptr) clamped[o] = clamp_bits;
}

template <bool BOUND, int CAM>
static decltype(&preprocess_kernel<BOUND, CAM, false>) preprocess_instance(bool da) {
  return da ? preprocess_kernel<BOUND, CAM, true> : preprocess_kernel<BOUND, CAM, false>;
}

void launch_preprocess(const gab200_forward_args& a, int views, const float* cameras, const float* tanfov,
                       SplatRec* rec, SplatAux* aux, uint32_t* tiles_touched, uint8_t* clamped, uint32_t* depth_keys,
                       uint32_t* ids, const DepthBuckets& buckets, uint32_t* tile_count, bool rec_depth,
                       cudaStream_t stream) {
  const int threads = PRE_NT, blocks = (a.P + threads - 1) / threads;
  if (blocks == 0) return;
  const int cam = cameras != nullptr ? CAM_TABLE : tanfov != nullptr ? CAM_DEVFOV : CAM_ARGS;
  auto kernel = a.input_mode == GAB200_INPUT_BOUND_RAW
                    ? (cam == CAM_TABLE    ? preprocess_instance<true, CAM_TABLE>(rec_depth)
                       : cam == CAM_DEVFOV ? preprocess_instance<true, CAM_DEVFOV>(rec_depth)
                                           : preprocess_instance<true, CAM_ARGS>(rec_depth))
                    : (cam == CAM_TABLE    ? preprocess_instance<false, CAM_TABLE>(rec_depth)
                       : cam == CAM_DEVFOV ? preprocess_instance<false, CAM_DEVFOV>(rec_depth)
                                           : preprocess_instance<false, CAM_ARGS>(rec_depth));
  launch_pdl(kernel, dim3(blocks, cameras != nullptr ? views : 1), threads, 0, stream, a, cameras, tanfov, rec, aux,
             tiles_touched, clamped, depth_keys, ids, a.exact_binning, buckets, tile_count);
}

// =====================================================================================================
// Per-splat depth sort as a bucket sort (design: binning.cu header).  preprocess_kernel has already counted the
// splats and instances of every bucket and given each splat its arrival rank.
//   depth_scatter_kernel : every CTA scans the bucket counts in shared memory, then scatters (key, id) of its
//                          splats to start[bucket] + rank.  CTA 0 also publishes the two exclusive prefixes and
//                          {N, M, overflow} in meta.
//   depth_bucket_kernel  : one CTA per bucket: ranks the bucket's (key, id) pairs by counting (they fit in shared
//                          memory; ~25 of them on average), writes the ids in (key, id) order -- the order of a
//                          stable sort by key of ids 0..P-1 -- and the running instance counts.
// =====================================================================================================
constexpr int DS_NT = 256;

// Exclusive prefix sum of s[0..n) in place (n a multiple of DS_NT); returns the total to every thread.  Warp w owns
// the contiguous slice [w n/8, (w+1) n/8) and walks it 32 elements at a time (lane = element: no bank conflicts --
// a thread-owns-a-run layout is a 32-way conflict on every access).
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t* s, int n, uint32_t* warp_tot) {
  constexpr unsigned FULL = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int slice = n / (DS_NT / 32);
  uint32_t carry = 0;
  for (int base = w * slice; base < (w + 1) * slice; base += 32) {
    const uint32_t v = s[base + lane];
    uint32_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t up = __shfl_up_sync(FULL, incl, d);
      if (lane >= d) incl += up;
    }
    s[base + lane] = carry + incl - v;
    carry += __shfl_sync(FULL, incl, 31);
  }
  if (lane == 0) warp_tot[w] = carry;
  __syncthreads();
  uint32_t wbase = 0, total = 0;
#pragma unroll
  for (int k = 0; k < DS_NT / 32; k++) {
    const uint32_t t = warp_tot[k];
    if (k < w) wbase += t;
    total += t;
  }
  for (int base = w * slice; base < (w + 1) * slice; base += 32) s[base + lane] += wbase;
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(DS_NT) depth_scatter_kernel(int P, DepthBuckets bk,
                                                              const uint32_t* __restrict__ depth_keys,
                                                              uint32_t* __restrict__ out_keys,
                                                              uint32_t* __restrict__ out_ids, uint32_t capacity,
                                                              uint32_t seq, uint32_t* __restrict__ sticky_overflow) {
  extern __shared__ uint32_t s_start[];  // [nb]
  __shared__ uint32_t warp_tot[DS_NT / 32];
  __shared__ uint32_t s_flag;
  const int tid = threadIdx.x, nb = (int)bk.nb;
  if (tid == 0) s_flag = 0;
  pdl_wait();
  pdl_trigger();
  uint32_t over = 0;
  for (int b = tid; b < nb; b += DS_NT) {
    const uint32_t c = bk.counts[b];
    s_start[b] = c;
    over |= (c > GAB_DEPTH_BUCKET_CAP) ? 1u : 0u;
  }
  __syncthreads();
  const uint32_t M = block_exclusive_scan(s_start, nb, warp_tot);
  if (blockIdx.x == 0) {
    if (over) atomicOr(&s_flag, 1u);
    for (int b = tid; b < nb; b += DS_NT) bk.start[b] = s_start[b];
  }
  const int i = blockIdx.x * DS_NT + tid;
  if (i < P) {
    const uint32_t key = depth_keys[i];
    if (key != 0xffffffffu) {
      const uint32_t pos = s_start[depth_bucket(key, bk)] + bk.rank[i];
      out_keys[pos] = key;
      out_ids[pos] = (uint32_t)i;
    }
  }
  if (blockIdx.x == 0) {  // second scan (instances per bucket), reusing the shared array
    __syncthreads();
    for (int b = tid; b < nb; b += DS_NT) s_start[b] = bk.tiles[b];
    __syncthreads();
    const uint32_t N = block_exclusive_scan(s_start, nb, warp_tot);
    for (int b = tid; b < nb; b += DS_NT) bk.tile_base[b] = s_start[b];
    if (tid == 0) {  // the frame counters of a bucket-sorted frame (publish_counters_kernel does this on the radix path)
      bk.meta[GAB200_CTR_NUM_RENDERED] = N;
      bk.meta[GAB200_CTR_NUM_LISTED] = M;
      bk.meta[GAB200_CTR_BUCKET_OVERFLOW] = s_flag;
      bk.meta[GAB200_CTR_CAPACITY] = capacity;
      bk.meta[GAB200_CTR_SEQ] = seq;
      const uint32_t hi = bk.meta[GAB_META_TOTAL64 + 1];
      bk.meta[GAB200_CTR_NUM_RENDERED_HI] = hi;
      if (sticky_overflow != nullptr && (hi != 0 || s_flag != 0 || N > capacity)) *sticky_overflow = 1u;
    }
  }
}

constexpr int DB_NT = 128;
__global__ void __launch_bounds__(DB_NT) depth_bucket_kernel(DepthBuckets bk, const uint32_t* __restrict__ keys,
                                                             uint32_t* __restrict__ ids_inout,
                                                             const uint32_t* __restrict__ tiles_touched,
                                                             uint32_t* __restrict__ offsets) {
  __shared__ unsigned long long comp[GAB_DEPTH_BUCKET_CAP];
  __shared__ uint32_t st[GAB_DEPTH_BUCKET_CAP];
  __shared__ uint32_t warp_tot[DB_NT / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  pdl_wait();
  pdl_trigger();
  const int n = (int)bk.counts[b];
  if (n == 0 || n > GAB_DEPTH_BUCKET_CAP) return;  // overflow: the host redoes the frame on the radix path
  const uint32_t start = bk.start[b], tbase = bk.tile_base[b];
  for (int j = tid; j < n; j += DB_NT)
    comp[j] = ((unsigned long long)keys[start + j] << 32) | (unsigned long long)ids_inout[start + j];
  __syncthreads();
  for (int t = tid; t < n; t += DB_NT) {
    const unsigned long long c = comp[t];
    int r = 0;
    for (int j = 0; j < n; j++) r += comp[j] < c ? 1 : 0;  // broadcast reads; ids are distinct -> ranks are too
    const uint32_t id = (uint32_t)c;
    ids_inout[start + r] = id;  // in place: the bucket's inputs are all in shared memory by now
    st[r] = tiles_touched[id];
  }
  __syncthreads();
  // inclusive running instance count in sorted order
  const int per = (n + DB_NT - 1) / DB_NT;
  const int j0 = min(tid * per, n), j1 = min(j0 + per, n);
  uint32_t local = 0;
  for (int j = j0; j < j1; j++) local += st[j];
  uint32_t incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t nbv = __shfl_up_sync(0xffffffffu, incl, d);
    if ((tid & 31) >= d) incl += nbv;
  }
  if ((tid & 31) == 31) warp_tot[tid >> 5] = incl;
  __syncthreads();
  uint32_t run = tbase + incl - local;
#pragma unroll
  for (int w = 0; w < DB_NT / 32; w++)
    if (w < (tid >> 5)) run += warp_tot[w];
  for (int j = j0; j < j1; j++) {
    run += st[j];
    offsets[start + j] = run;
  }
}

void launch_depth_bucket_sort(int P, const DepthBuckets& bk, const uint32_t* depth_keys, const uint32_t* tiles_touched,
                              uint32_t* scratch_keys, uint32_t* sorted_ids, uint32_t* offsets, uint32_t capacity,
                              uint32_t seq, uint32_t* sticky_overflow, cudaStream_t stream) {
  if (P <= 0) return;
  launch_pdl(depth_scatter_kernel, (P + DS_NT - 1) / DS_NT, DS_NT, bk.nb * sizeof(uint32_t), stream, P, bk, depth_keys,
             scratch_keys, sorted_ids, capacity, seq, sticky_overflow);
  launch_pdl(depth_bucket_kernel, bk.nb, DB_NT, 0, stream, bk, scratch_keys, sorted_ids, tiles_touched, offsets);
}

// =====================================================================================================
// Export of the binding + activation only (gab200_bind_activate)
// =====================================================================================================
__global__ void __launch_bounds__(256) bind_activate_kernel(gab200_forward_args a, float* __restrict__ means3D,
                                                            float* __restrict__ opacities,
                                                            float* __restrict__ scales, float* __restrict__ cov3D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  Activated act;
  bind_activate(a, i, act);
  if (means3D) {
    means3D[3 * (size_t)i] = act.mean.x;
    means3D[3 * (size_t)i + 1] = act.mean.y;
    means3D[3 * (size_t)i + 2] = act.mean.z;
  }
  if (opacities) opacities[i] = act.opacity;
  if (scales) {
    scales[3 * (size_t)i] = act.s[0];
    scales[3 * (size_t)i + 1] = act.s[1];
    scales[3 * (size_t)i + 2] = act.s[2];
  }
  if (cov3D) {
    float s[3] = {a.scale_modifier * act.s[0], a.scale_modifier * act.s[1], a.scale_modifier * act.s[2]};
    float c3[6];
    cov3d_from_R(act.R, s, c3);
#pragma unroll
    for (int k = 0; k < 6; k++) cov3D[6 * (size_t)i + k] = c3[k];
  }
}

void launch_bind_activate(const gab200_forward_args& a, float* means3D, float* opacities, float* scales, float* cov3D,
                          cudaStream_t stream) {
  const int threads = 256, blocks = (a.P + threads - 1) / threads;
  if (blocks == 0) return;
  bind_activate_kernel<<<blocks, threads, 0, stream>>>(a, means3D, opacities, scales, cov3D);
  count_launch();
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ V,
                                    uint8_t* __restrict__ present) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float3 p = make_float3(means3D[3 * (size_t)i], means3D[3 * (size_t)i + 1], means3D[3 * (size_t)i + 2]);
  float z = V[2] * p.x + V[6] * p.y + V[10] * p.z + V[14];
  present[i] = z > 0.2f ? 1 : 0;
}

void launch_mark_visible(int P, const float* means3D, const float* V, uint8_t* present, cudaStream_t stream) {
  if (P == 0) return;
  mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, V, present);
  count_launch();
}

// =====================================================================================================
// K3: tile|depth key emission.  Emission order inside a splat is row-major (y, then x) from offsets[i-1] --
// identical to the reference, so the stable sort's tie order is too.
//   exact list  : one WARP per 32 splats, lanes cooperate on each splat's rectangle (a 1000-tile splat does not
//                 serialise one thread; stores coalesce).
//   culled list : one THREAD per splat walks its rows (a few sqrt per row, ~4 rows on average); splats with many
//                 rows are handed to the whole warp afterwards, one row per lane.
// =====================================================================================================
#define EMIT_HEAVY_ROWS 12

// VIEWS (gab200_forward_views): splat i of the depth order is virtual splat view * view_splats + local; its instances
// go to the tiles view * view_tiles + the tile in the view.
// The clears the radix tile sort needs before it, done by the emission grid instead of memset nodes on the frame's
// stream (each such node is a boundary of its own, and a kernel behind a memset cannot launch early): the ranges
// [0, n_ranges), the block masks [0, n_mask) (16-B stores: the binning buffer's slack covers the round-up) and, with
// `sentinel` (count only on the device), the padding keys [n, cap) behind the n = min(N, cap) instances the emission
// writes -- all cap keys when a depth bucket overflowed and nothing is emitted.
__device__ __forceinline__ void emit_clears(const uint32_t* counters, const uint32_t* order_count, uint32_t cap,
                                            uint32_t* keys, bool sentinel, uint8_t* mask, uint32_t n_mask,
                                            uint2* ranges, uint32_t n_ranges) {
  const uint32_t stride = gridDim.x * blockDim.x, t = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t j = t; j < n_ranges; j += stride) ranges[j] = make_uint2(0u, 0u);
  if (mask != nullptr)
    for (uint32_t j = t; j < (n_mask + 15u) / 16u; j += stride) reinterpret_cast<uint4*>(mask)[j] = make_uint4(0, 0, 0, 0);
  if (sentinel) {
    uint32_t n = counters[GAB200_CTR_NUM_RENDERED_HI] != 0 ? cap : min(counters[GAB200_CTR_NUM_RENDERED], cap);
    if (order_count != nullptr && counters[GAB200_CTR_BUCKET_OVERFLOW] != 0) n = 0;
    for (uint32_t j = n + t; j < cap; j += stride) keys[j] = 0xffffffffu;
  }
}

template <bool VIEWS>
__device__ __forceinline__ void emit_keys(int P, int gx, int gy, const SplatRec* rec, const SplatAux* aux,
                                          const uint32_t* order, const uint32_t* offsets, const uint32_t* order_count,
                                          const uint32_t* counters, uint32_t cap, uint32_t* cursor, uint32_t* keys,
                                          uint32_t* vals, int exact_binning, uint32_t view_splats, uint32_t view_tiles) {
  constexpr unsigned FULL = 0xffffffffu;
  // cursor != nullptr (counting tile sort): an instance goes to the next free slot of ITS TILE's segment and carries
  // the splat's depth rank as key; otherwise it goes to offsets[...] + k in emission order with the tile id as key
  // (input of the stable radix sort by tile).
  auto put = [&](uint32_t o, uint32_t tile, uint32_t rank, uint32_t id) {
    if (cursor != nullptr) {
      o = atomicAdd(cursor + tile, 1u);
      tile = rank;
    }
    if (o < cap) {
      keys[o] = tile;
      vals[o] = id;
    }
  };
  // a depth bucket overflowed: `order` / `offsets` are incomplete, the host (or the graph's owner) redoes the frame
  if (order_count != nullptr && counters[GAB200_CTR_BUCKET_OVERFLOW] != 0) return;
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int slot = warp_global * 32 + lane;  // position in DEPTH order; the splat it holds is order[slot]
  float px = 0.f, py = 0.f, cA = 0.f, cB = 0.f, cC = 0.f, op = 0.f;
  int radius = 0;
  uint32_t ntiles = 0, off = 0, i = 0, tb = 0;  // tb: first tile of the splat's view
  // bucket-sorted frames list only the M splats that emit instances; radix-sorted frames list all P (culled last)
  const int listed = order_count != nullptr ? (int)*order_count : P;
  if (slot < listed) {
    i = order[slot];
    const SplatAux ax = aux[i];
    ntiles = ax.tiles;
    if (ntiles) {
      const float4 q0 = rec[i].q0;
      const float4 q1 = rec[i].q1;
      px = q0.x; py = q0.y; op = q1.y;
      cA = q0.z / REC_SCALE_AC; cB = q0.w / REC_SCALE_B; cC = q1.x / REC_SCALE_AC;  // undo the blend pre-scale
      radius = ax.radius;
      off = (slot == 0 || offsets == nullptr) ? 0u : offsets[slot - 1];
      if (VIEWS) tb = (i / view_splats) * view_tiles;
    }
  }
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  if (ntiles) tile_rect(px, py, radius, gx, gy, x0, y0, x1, y1);

  if (exact_binning) {
    uint32_t todo = __ballot_sync(FULL, ntiles != 0);
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const int sx0 = __shfl_sync(FULL, x0, src), sy0 = __shfl_sync(FULL, y0, src);
      const int w = __shfl_sync(FULL, x1, src) - sx0;
      const int cnt = (int)__shfl_sync(FULL, ntiles, src);
      const uint32_t soff = __shfl_sync(FULL, off, src);
      const uint32_t sid = __shfl_sync(FULL, i, src);
      const uint32_t stb = VIEWS ? __shfl_sync(FULL, tb, src) : 0u;
      for (int t = lane; t < cnt; t += 32) {
        const int y = sy0 + t / w, x = sx0 + t % w;
        put(soff + t, stb + (uint32_t)(y * gx + x), (uint32_t)(warp_global * 32 + src), sid);
      }
    }
    return;
  }

  // ---- culled list ----
  const bool heavy = ntiles != 0 && (y1 - y0) > EMIT_HEAVY_ROWS;
  if (ntiles != 0 && !heavy) {
    TileSpan span(px, py, cA, cB, cC, op, x0, x1);
    uint32_t o = off;
    for (int ty = y0; ty < y1; ty++) {
      int cx0, cx1;
      span.row(ty, cx0, cx1);
      for (int x = cx0; x < cx1; x++) {
        put(o, tb + (uint32_t)(ty * gx + x), (uint32_t)slot, i);
        o++;
      }
    }
  }
  uint32_t todo = __ballot_sync(FULL, heavy);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const float spx = __shfl_sync(FULL, px, src), spy = __shfl_sync(FULL, py, src);
    const float sA = __shfl_sync(FULL, cA, src), sB = __shfl_sync(FULL, cB, src), sC = __shfl_sync(FULL, cC, src);
    const float sop = __shfl_sync(FULL, op, src);
    const int sx0 = __shfl_sync(FULL, x0, src), sx1 = __shfl_sync(FULL, x1, src);
    const int sy0 = __shfl_sync(FULL, y0, src), sy1 = __shfl_sync(FULL, y1, src);
    uint32_t base = __shfl_sync(FULL, off, src);
    const uint32_t sid = __shfl_sync(FULL, i, src);
    const uint32_t stb = VIEWS ? __shfl_sync(FULL, tb, src) : 0u;
    TileSpan span(spx, spy, sA, sB, sC, sop, sx0, sx1);
    for (int r0 = sy0; r0 < sy1; r0 += 32) {  // 32 rows at a time: lane = row
      const int ty = r0 + lane;
      int cx0 = 0, cx1 = 0;
      if (ty < sy1) span.row(ty, cx0, cx1);
      const int len = cx1 - cx0;
      int incl = len;  // warp inclusive scan of the row lengths -> each row's offset
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int nb = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += nb;
      }
      uint32_t o = base + (uint32_t)(incl - len);
      for (int x = cx0; x < cx1; x++) {
        put(o, stb + (uint32_t)(ty * gx + x), (uint32_t)(warp_global * 32 + src), sid);
        o++;
      }
      base += (uint32_t)__shfl_sync(FULL, incl, 31);
    }
  }
}

template <bool VIEWS>
__global__ void __launch_bounds__(256) emit_keys_kernel(int P, int gx, int gy, const SplatRec* __restrict__ rec,
                                                        const SplatAux* __restrict__ aux,
                                                        const uint32_t* __restrict__ order,
                                                        const uint32_t* __restrict__ offsets,
                                                        const uint32_t* __restrict__ order_count,
                                                        const uint32_t* __restrict__ counters, uint32_t cap,
                                                        uint32_t* __restrict__ cursor,
                                                        uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                        int exact_binning, uint32_t view_splats, uint32_t view_tiles,
                                                        bool sentinel, uint8_t* __restrict__ mask, uint32_t n_mask,
                                                        uint2* __restrict__ ranges, uint32_t n_ranges) {
  pdl_wait();
  pdl_trigger();
  emit_clears(counters, order_count, cap, keys, sentinel, mask, n_mask, ranges, n_ranges);
  emit_keys<VIEWS>(P, gx, gy, rec, aux, order, offsets, order_count, counters, cap, cursor, keys, vals, exact_binning,
                   view_splats, view_tiles);
}

__global__ void publish_counters_kernel(uint32_t* __restrict__ counters, const uint32_t* __restrict__ offsets, int P,
                                        uint32_t capacity, uint32_t seq, uint32_t* __restrict__ sticky_overflow) {
  pdl_wait();
  pdl_trigger();
  if (P > 0) {  // radix-sorted frame: every splat is listed; N is the last inclusive offset (unless already counted)
    if (offsets != nullptr) counters[GAB200_CTR_NUM_RENDERED] = offsets[P - 1];
    counters[GAB200_CTR_NUM_LISTED] = (uint32_t)P;
    counters[GAB200_CTR_BUCKET_OVERFLOW] = 0;
  }
  counters[GAB200_CTR_CAPACITY] = capacity;
  counters[GAB200_CTR_SEQ] = seq;
  const uint32_t hi = counters[GAB_META_TOTAL64 + 1];
  counters[GAB200_CTR_NUM_RENDERED_HI] = hi;
  if (sticky_overflow != nullptr &&
      (hi != 0 || counters[GAB200_CTR_BUCKET_OVERFLOW] != 0 || counters[GAB200_CTR_NUM_RENDERED] > capacity))
    *sticky_overflow = 1u;
}
void launch_publish_counters(uint32_t* counters, const uint32_t* offsets, int P, uint32_t capacity, uint32_t seq,
                             uint32_t* sticky_overflow, cudaStream_t stream) {
  launch_pdl(publish_counters_kernel, 1, 1, 0, stream, counters, offsets, P, capacity, seq, sticky_overflow);
}

void launch_emit_keys(int P, int gx, int gy, const SplatRec* rec, const SplatAux* aux, const uint32_t* order,
                      const uint32_t* offsets, const uint32_t* order_count, const uint32_t* counters, uint32_t cap,
                      uint32_t* cursor, uint32_t* keys, uint32_t* vals, int exact_binning, int view_splats,
                      const EmitClears& clr, cudaStream_t stream) {
  const int warps = (P + 31) / 32;
  const int threads = 256, blocks = (warps * 32 + threads - 1) / threads;
  if (blocks == 0) return;
  launch_pdl(view_splats > 0 ? emit_keys_kernel<true> : emit_keys_kernel<false>, blocks, threads, 0, stream, P, gx, gy,
             rec, aux, order, offsets, order_count, counters, cap, cursor, keys, vals, exact_binning,
             (uint32_t)view_splats, (uint32_t)(gx * gy), clr.sentinel, clr.mask, clr.n_mask, clr.ranges, clr.n_ranges);
}

// =====================================================================================================
// K5: tile ranges from key transitions in the sorted stream (ranges zeroed by the emission, EmitClears).
// =====================================================================================================
// Keys >= tiles are the padding of a capacity-sized sort (sentinel 0xffffffff): they sort behind every real instance
// and all of them land in the spare slot ranges[tiles], which nobody reads.
__global__ void __launch_bounds__(256) tile_ranges_kernel(int64_t N, uint32_t tiles, const uint32_t* __restrict__ keys,
                                                          uint2* __restrict__ ranges) {
  pdl_wait();
  pdl_trigger();
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N) return;
  const uint32_t cur = min(keys[idx], tiles);
  if (idx == 0)
    ranges[cur].x = 0;
  else {
    const uint32_t prev = min(keys[idx - 1], tiles);
    if (cur != prev) {
      ranges[prev].y = (uint32_t)idx;
      ranges[cur].x = (uint32_t)idx;
    }
  }
  if (idx == N - 1) ranges[cur].y = (uint32_t)N;
}

__global__ void expand_keys_kernel(int64_t N, const uint32_t* __restrict__ tile_keys, const uint32_t* __restrict__ ids,
                                   const SplatAux* __restrict__ aux, uint64_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  out[i] = ((uint64_t)tile_keys[i] << 32) | (uint64_t)__float_as_uint(aux[ids[i]].depth);
}
// the reference's key format (tile << 32 | fp32 depth bits) rebuilt from the two-stage sort's outputs (parity export)
void launch_expand_keys(int64_t N, const uint32_t* tile_keys, const uint32_t* ids, const SplatAux* aux, uint64_t* out,
                        cudaStream_t stream) {
  if (N == 0) return;
  expand_keys_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(N, tile_keys, ids, aux, out);
  count_launch();
}

void launch_tile_ranges(int64_t N, uint32_t tiles, const uint32_t* keys, uint2* ranges, cudaStream_t stream) {
  if (N == 0) return;
  const int threads = 256;
  const int64_t blocks = (N + threads - 1) / threads;
  launch_pdl(tile_ranges_kernel, (unsigned)blocks, threads, 0, stream, N, tiles, keys, ranges);
}

}  // namespace gab
