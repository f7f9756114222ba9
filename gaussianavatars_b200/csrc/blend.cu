// blend.cu -- per-tile front-to-back alpha blend (forward) and reverse-walk gradient (backward) for sm_90a.
// Replaces renderCUDA fwd/bwd of the reference module (SURVEY.md 2.4 K6/K7, Appendix B.3/B.4).
//
// Mapping (NOT the reference's 1 thread = 1 pixel, 256-thread block for every tile):
//   * BANDS: a 16x16 tile is 2 halves (8 columns) x 4 bands (4 rows) = eight 8x4-pixel blocks.  A warp owns one
//     half and K bands of it; lane = (column 0..7, row-in-band 0..3) and owns the K pixels (column, 4 b + row) of its
//     bands.  The x-offset to a splat (dx) is shared by a lane's K pixels, so the exponent costs 3 flops per pixel,
//         power(dy) = p0 + dy * (q + h * dy),   p0 = -A dx^2/2, q = -B dx, h = -C/2   (pre-scaled by log2 e -> ex2),
//     the shared-memory broadcast reads of the splat record are amortised K times, and every instruction of a band
//     covers a COMPACT 8x4 block: a splat either touches most of its lanes or none (a 16x2 strip, the round-1 shape,
//     ran its gradient code with 18 of 32 lanes live).
//   * HYBRID TILE SCHEDULE: the tiles are launched heaviest-first (tile_order_kernel).  A CTA takes either ONE heavy
//     tile with many warps and few pixels per thread (short per-warp critical path for 2000-deep lists) or SEVERAL
//     light tiles, each on a 64-thread group with K = 4 (fewest instructions); groups synchronise on their own
//     named barrier.  A uniform K = 4 leaves the SMs idle waiting for a few deep tiles; a uniform K = 1 is
//     issue-bound.
//   * splat records (48 B, three 16-B quads) are GATHERED straight into shared memory with cp.async (LDGSTS),
//     double buffered one chunk ahead, ids one further chunk ahead: no register staging, no exposed L2 latency.
//   * forward: per 32-splat group, each warp tests the splats' alpha boxes against its pixels (reaches_rect) and walks
//     only the live ones, through a per-warp list of their offsets.
//   * forward records, per sorted instance, which of the tile's eight 8x4 blocks it contributed to (one byte);
//     backward visits a (splat, warp) pair only if one of the warp's blocks is set.
//   * backward: one WARP task per (tile, half, band group) -- K = 2 on heavy tiles, K = 4 on light ones -- with a
//     private TMA ring for its id/mask lists and no CTA barrier.  A visit with all K bands live is straight-line code
//     in which the bands' dependency chains interleave (ILP); otherwise the live bands run under warp-uniform
//     branches and dead bands cost nothing.  Lanes whose pixel did not contribute carry alpha = G = 0 through the
//     same instructions (no divergence).  Per-lane partial sums over the K pixels collapse to three moments
//     (S0,S1,S2) because dx is shared, and the nine per-splat gradient components of three consecutive visits leave
//     together through a shared-memory row reduction that ends in one 27-lane RED.ADD.F32 per three visits.
// Tensor cores are not used: there is no dense contraction on this path (north_star).
#include <type_traits>

#include "common.cuh"
#include "kernels.cuh"

namespace gab {

#define LOG2E 1.4426950408889634f
#define ALPHA_MIN (1.0f / 255.0f)
#define FULLMASK 0xffffffffu
// SplatRec stores the conic pre-scaled for the exponent in log2 units: (A',B',C') = (-A/2, -B, -C/2) * log2(e)
#define CONIC_UNSCALE_AC (-2.0f / LOG2E)
#define CONIC_UNSCALE_B (-1.0f / LOG2E)

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void gather_rec(SplatRec* dst, const SplatRec* src) {
  cp_async16(&dst->q0, &src->q0);
  cp_async16(&dst->q1, &src->q1);
  cp_async16(&dst->q2, &src->q2);
}

// ---- TMA bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier: the per-tile splat-id lists are contiguous runs of the
// sorted stream, so they are brought into shared memory by the copy engine, NT ids per transaction, two chunks
// ahead of the blend, without occupying LSU slots or registers.  (The 48-B records those ids point at are a gather
// and stay on cp.async.)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tMBAR_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra MBAR_DONE;\n\t"
      "bra MBAR_WAIT;\n\tMBAR_DONE:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
#define GAB_FWD_DEPTH_CTAS 2  // CTAs per SM the depth-plane blend kernels are bounded for (DESIGN.md section 4)
#define GAB_FWD_VIEWS_TRAIN_CTAS 3  // ... and the K-view training forward
#define GAB_BWD_DEPTH_CTAS 5
#define ID_RING 3  // id chunks in flight: being gathered from, next, and the one the copy engine is filling

// Barrier of one thread group (NT threads, hardware barrier `id`); id 0 with NT = blockDim is __syncthreads().
template <int NT>
struct GroupBarrier {
  int id;
  __device__ __forceinline__ void sync() const { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(NT) : "memory"); }
  __device__ __forceinline__ bool sync_and(bool pred) const {
    unsigned r;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %1, 0;\n\tbar.red.and.pred p, %2, %3, q;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(r)
        : "r"((unsigned)pred), "r"(id), "n"(NT)
        : "memory");
    return r != 0;
  }
};

// Pixel ownership inside a 16x16 tile for a group of 256/K threads (thread tl): warp w = tl/32 owns half h = w & 1
// (columns 8h .. 8h+7) and the K bands (w/2) K .. (w/2) K + K-1 (band b = rows 4b .. 4b+3); lane = (column, row in
// band).  bit(i) = position of block (h, band i of this warp) in the per-instance block mask byte.
template <int K>
struct BandGeom {
  int col, row0, half, band0;
  __device__ __forceinline__ explicit BandGeom(int tl) {
    const int w = tl >> 5, lane = tl & 31;
    half = w & 1;
    band0 = (w >> 1) * K;
    col = half * 8 + (lane & 7);
    row0 = band0 * 4 + (lane >> 3);
  }
  __device__ __forceinline__ int bit(int i) const { return 2 * (band0 + i) + half; }
};

// ---- display epilogue: the image as interleaved uint8 [H,W,3], quantised as render.py:41 does it,
// data.mul(255).add_(0.5).clamp_(0, 255) then the cast (truncation).  The multiply and the add are separately rounded
// (no contraction into an fma), so the byte equals torch's two ops on the float the float path stores, bit for bit.
#define BLEND_OUT_FLOAT 1  // [3,H,W] float32
#define BLEND_OUT_U8 2     // [H,W,3] uint8
#define BLEND_OUT_TRAIN 4  // final_T and n_contrib [H,W] and the block masks, which the backward reads
#define BLEND_OUT_VIEWER 8 // with BLEND_OUT_U8: the display bytes quantised as the local viewer's export does
__device__ __forceinline__ uint32_t quantize_u8(float c) {
  return __float2uint_rz(fminf(fmaxf(__fadd_rn(__fmul_rn(c, 255.f), 0.5f), 0.f), 255.f));
}
// One row of a band is 8 lanes (lane = row * 8 + column) holding 8 consecutive pixels: 24 bytes = 6 words.  Lane
// (row, j < 6) writes word j, bytes 4j .. 4j+3, which lie in pixels p0 = 4j/3 and p0 + 1 from byte 4j - 3 p0 of p0:
// two shuffles per band, and the warp stores whole aligned 32-bit words instead of 96 scattered bytes.  A row whose
// start is not word-aligned (W % 4 != 0) or that the image's right edge cuts stores bytes.  All 32 lanes call this.
// VIEWER: quantize_u8_viewer in place of quantize_u8 (GAB200_QUANTIZE_VIEWER).
template <bool VIEWER>
__device__ __forceinline__ void store_display(uint8_t* __restrict__ out, int W, int H, int pixx, int y, int lane,
                                              float r, float g, float b) {
  const uint32_t px = VIEWER ? quantize_u8_viewer(r) | (quantize_u8_viewer(g) << 8) | (quantize_u8_viewer(b) << 16)
                             : quantize_u8(r) | (quantize_u8(g) << 8) | (quantize_u8(b) << 16);
  const int j = lane & 7, x0 = pixx - j;
  const int p0 = min((4 * j) / 3, 6);
  const uint32_t lo = __shfl_sync(FULLMASK, px, (lane & ~7) | p0);
  const uint32_t hi = __shfl_sync(FULLMASK, px, (lane & ~7) | (p0 + 1));
  const uint32_t word = (uint32_t)((((uint64_t)hi << 24) | lo) >> (8 * (4 * j - 3 * p0)));
  if (y >= H) return;
  const size_t row = (size_t)y * W;
  if ((W & 3) == 0 && x0 + 8 <= W && ((uintptr_t)out & 3u) == 0) {
    if (j < 6) reinterpret_cast<uint32_t*>(out)[(row + x0) / 4 * 3 + j] = word;
  } else if (pixx < W) {
    uint8_t* o = out + (row + pixx) * 3;
    o[0] = (uint8_t)px;
    o[1] = (uint8_t)(px >> 8);
    o[2] = (uint8_t)(px >> 16);
  }
}

// Can splat r reach alpha >= 1/255 at a pixel centre of the rectangle [x0, x1] x [y0, y1]?  The test of the splat's
// alpha box against the rectangle: (rx, ry) = q2.yz are TileSpan's extents of the ellipse
//   q(d) = 1/2 (A dx^2 + C dy^2) + B dx dy <= tau = ln(255 opacity) + 0.01,   rx = sqrt(2 tau C / det) + 0.02 px
// (ry likewise with A), 1e30 for a degenerate conic and -1 when tau <= 0 (no alpha reaches 1/255: never live).  A
// NaN centre or extent counts as live.
// Why a skipped splat is one the unculled walk would not have changed anything for: a pixel centre outside the box
// lies outside the ellipse q = tau, so its exact alpha is below e^-0.01 / 255 = 0.990 / 255.  The walk computes pw in
// float (two fmaf and a product, rounding error at most ~4 ulp of the largest term |A'| dx^2, |B' dx dy|, |C'| dy^2,
// whose sum is at most (kappa + 1) |pw| for a conic of condition number kappa), ex2.approx.ftz (relative error below
// 2^-22, PTX ISA) and op * G, and accepts alpha >= 1/255.  Accepting a pixel whose exact alpha is below 0.990 / 255
// takes an error of 0.0144 in pw (the 0.01 log margin in log2 units); with |pw| <= 8 near the boundary, the rounding
// stays below that for kappa up to ~7e3, and ex2's error is five orders of magnitude short of it.  The +0.02 px
// margin adds 2 tau 0.02 / rx to q at the box edge on top.  Such a pixel fails `pw <= 0 && alpha >= 1/255` in the
// walk: no T, colour, depth, `done`, `last` or block-mask bit changes, so skipping the splat for the whole warp leaves
// every output bit-identical.  The binning (TileSpan::row) drops whole tiles on the same margins; this test applies
// them to the warp's 8x4 blocks.  tests/test_gpu_forward_cull.py checks the claim in float32 on the adversarial rigs.
__device__ __forceinline__ bool reaches_rect(const SplatRec& r, float x0, float x1, float y0, float y1) {
  const float4 q0 = r.q0, q2 = r.q2;
  const float ex = fmaxf(fmaxf(x0 - q0.x, q0.x - x1), 0.f);  // distance from the centre to the rectangle, per axis
  const float ey = fmaxf(fmaxf(y0 - q0.y, q0.y - y1), 0.f);
  return !(ex > q2.y) && !(ey > q2.z);
}

// =====================================================================================================
// Forward: one tile on a group of NT = 256/K threads (tl = thread index inside the group)
// =====================================================================================================
// OUT: which images are written (BLEND_OUT_*).  Without BLEND_OUT_TRAIN the training outputs (final_T, n_contrib and
// the block masks) are absent at compile time; with it they are written where final_T / strip_mask are non-null.
// DA (gab200_forward*_depth_alpha): also the accumulated alpha 1 - T_final and the depth sum_i w_i z_i of the same
// walk, z_i = q2.w of a record written by the preprocess with DA; out_alpha / out_depth [H,W] (either may be NULL).
// VIEWS (gab200_forward_views*): `tile` is global tile g of K views, tile g % view_tiles of view g / view_tiles: the
// tile's range and the view's per-pixel outputs are offset by view, then the tile is rendered exactly as a single
// view.  The block masks are indexed by position in the sorted stream, which is global already.
template <int K, int OUT, bool DA, bool VIEWS>
__device__ __forceinline__ void forward_tile(int tile, int tl, GroupBarrier<256 / K> bar, SplatRec* buf0,
                                             SplatRec* buf1, uint32_t* smask, uint32_t* ids_ring, uint64_t* mbar,
                                             int W, int H, int gx, int view_tiles,
                                             const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                                             const SplatRec* __restrict__ rec, const float* __restrict__ bg,
                                             float* __restrict__ out_color, float* __restrict__ final_T,
                                             uint32_t* __restrict__ n_contrib, uint8_t* __restrict__ strip_mask,
                                             uint8_t* __restrict__ out_rgb8, float* __restrict__ out_alpha,
                                             float* __restrict__ out_depth) {
  constexpr bool TRAIN = DA || (OUT & BLEND_OUT_TRAIN) != 0;
  if (VIEWS) {
    const int view = tile / view_tiles;
    const size_t off = (size_t)view * H * W;
    tile -= view * view_tiles;
    ranges += (size_t)view * view_tiles;
    if (OUT & BLEND_OUT_FLOAT) out_color += 3 * off;
    if (OUT & BLEND_OUT_U8) out_rgb8 += 3 * off;
    if (TRAIN && final_T != nullptr) {
      final_T += off;
      n_contrib += off;
    }
    if (DA && out_alpha != nullptr) out_alpha += off;
    if (DA && out_depth != nullptr) out_depth += off;
  }
  constexpr int NT = 256 / K;
  const int tx = tile % gx, ty = tile / gx;
  const int lane = tl & 31;
  const BandGeom<K> geo(tl);
  const int pixx = tx * GAB_TILE + geo.col;
  const int pixy0 = ty * GAB_TILE + geo.row0;  // the lane's pixel of band i is (pixx, pixy0 + 4 i)
  const float fx = (float)pixx;
  float fy[K];  // pixel rows as floats: dy = py - fy[i] is then independent of K (same bits on every tile schedule)
#pragma unroll
  for (int i = 0; i < K; i++) fy[i] = (float)(pixy0 + 4 * i);
  const uint2 range = ranges[tile];
  const int n = (int)(range.y - range.x);
  const uint32_t* ids = point_list + range.x;
  const bool want_mask = TRAIN && strip_mask != nullptr;
  smask[tl] = 0;
  // the warp's pixel rectangle: columns of its half, rows of its K bands (pixels past the image edge included)
  const float rx0 = (float)(pixx - (lane & 7)), rx1 = rx0 + 7.f;
  const float ry0 = (float)(ty * GAB_TILE + geo.band0 * 4), ry1 = ry0 + (float)(4 * K - 1);
  __shared__ uint8_t live_idx[8][32];  // per warp of the CTA: the group offsets of the live splats, in list order
  uint8_t* my_idx = live_idx[threadIdx.x >> 5];

  float T[K], Cr[K], Cg[K], Cb[K];
  float D[DA ? K : 1];
  uint32_t last[K];
  uint32_t done = 0;
  constexpr uint32_t ALL = (1u << K) - 1u;
#pragma unroll
  for (int i = 0; i < K; i++) {
    T[i] = 1.f; Cr[i] = Cg[i] = Cb[i] = 0.f; last[i] = 0;
    if (DA) D[i] = 0.f;
    if (pixx >= W || pixy0 + 4 * i >= H) done |= 1u << i;
  }

  const int nchunks = (n + NT - 1) / NT;
  // ---- id pipeline: chunk k of the tile's id list -> ids_ring[k % ID_RING] by one bulk copy (TMA), completion on
  // mbar[k % ID_RING].  Bulk copies need 16-B aligned addresses and sizes: the run starts at any 4-B offset, so the
  // copy starts `mis` ids early and carries 4 extra ids (the surplus is never read; it stays inside the binning buffer).
  constexpr int RING_STRIDE = NT + 4;
  constexpr uint32_t CHUNK_BYTES = RING_STRIDE * 4;
  const int mis = (int)(range.x & 3u);
  const uint32_t* ids_al = ids - mis;
  if (tl == 0) {
#pragma unroll
    for (int k = 0; k < ID_RING; k++) mbar_init(&mbar[k], 1);
    mbar_fence_init();
  }
  bar.sync();
  auto issue_ids = [&](int k) {  // one thread: arm the barrier with the byte count, start the copy
    uint64_t* b = &mbar[k % ID_RING];
    mbar_arrive_expect_tx(b, CHUNK_BYTES);
    bulk_copy_g2s(ids_ring + (k % ID_RING) * RING_STRIDE, ids_al + (size_t)k * NT, CHUNK_BYTES, b);
  };
  auto wait_ids = [&](int k) { mbar_wait(&mbar[k % ID_RING], (uint32_t)((k / ID_RING) & 1)); };
  if (tl == 0) {
    if (nchunks > 0) issue_ids(0);
    if (nchunks > 1) issue_ids(1);
  }
  // prologue: gather the records of chunk 0
  if (nchunks > 0) {
    wait_ids(0);
    if (tl < n) gather_rec(&buf0[tl], rec + ids_ring[mis + tl]);
  }
  cp_async_commit();

  for (int c = 0; c < nchunks; c++) {
    SplatRec* nxt = ((c + 1) & 1) ? buf1 : buf0;
    if (c + 1 < nchunks) {  // records of chunk c+1 (its ids arrived while chunk c-1 was blended)
      wait_ids(c + 1);
      const int p = (c + 1) * NT + tl;
      if (p < n) gather_rec(&nxt[tl], rec + ids_ring[((c + 1) % ID_RING) * RING_STRIDE + mis + tl]);
    }
    cp_async_commit();
    // ids of chunk c+2: its ring slot was last read (chunk c-1) before the group barrier that closed iteration c-1
    if (tl == 0 && c + 2 < nchunks) issue_ids(c + 2);
    cp_async_wait<1>();
    if (bar.sync_and(done == ALL)) {       // also publishes chunk c to the group
      if (c + 2 < nchunks) wait_ids(c + 2);  // never leave with a bulk copy still landing in our shared memory
      break;
    }
    const SplatRec* cur = (c & 1) ? buf1 : buf0;
    const int cnt = min(NT, n - c * NT);
    const uint32_t pos0 = (uint32_t)(c * NT);
    // Block bookkeeping for the backward pass, ~2 instructions per splat: every lane records, one bit per splat of
    // the current 32-splat group, whether its pixel of band i contributed; at the end of the group one REDUX.OR per
    // band turns the lanes' words into "block (half, band i) was touched by splat gbase+L" and lane L publishes splat L.
    uint32_t lb[K];
#pragma unroll
    for (int i = 0; i < K; i++) lb[i] = 0;
    // 32-splat groups: lane L first tests splat gbase+L against the warp's rectangle (reaches_rect) and the ballot's
    // set bits are compacted into a list of group offsets, so the inner loop walks only those splats, branch-light
    // and unrolled, with every record address independent of the previous iteration; the per-group epilogue
    // publishes the strip bits and tests saturation once per group.
    for (int gbase = 0; gbase < cnt; gbase += 32) {
      const int gend = min(32, cnt - gbase);
      const uint32_t live = __ballot_sync(FULLMASK, lane < gend && reaches_rect(cur[gbase + lane], rx0, rx1, ry0, ry1));
      const int nlive = __popc(live);
      __syncwarp();  // the previous group's walk has read the list
      if ((live >> lane) & 1u) my_idx[__popc(live & ((1u << lane) - 1u))] = (uint8_t)lane;
      __syncwarp();
#pragma unroll 4
      for (int k = 0; k < nlive; k++) {
        const int jj = my_idx[k];
        const SplatRec* r = cur + gbase + jj;
        const float4 q0 = r->q0;
        const float4 q1 = r->q1;
        const float dx = q0.x - fx;
        const float tA = q0.z * dx;  // conic pre-scaled by preprocess: pw = A' dx^2 + B' dx dy + C' dy^2 (log2 units)
#pragma unroll
        for (int i = 0; i < K; i++) {
          const float dy = q0.y - fy[i];
          const float pw = fmaf(q1.x * dy, dy, fmaf(q0.w, dy, tA) * dx);
          const float alpha = fminf(0.99f, q1.y * ex2_approx(pw));
          if (pw <= 0.f && alpha >= ALPHA_MIN && !((done >> i) & 1u)) {
            const float test_T = T[i] * (1.f - alpha);
            if (test_T < 0.0001f) {
              done |= 1u << i;
            } else {
              const float w = alpha * T[i];
              Cr[i] = fmaf(q1.z, w, Cr[i]);
              Cg[i] = fmaf(q1.w, w, Cg[i]);
              Cb[i] = fmaf(r->q2.x, w, Cb[i]);
              if (DA) D[i] = fmaf(r->q2.w, w, D[i]);
              T[i] = test_T;
              last[i] = pos0 + (uint32_t)(gbase + jj) + 1u;
              lb[i] |= 1u << jj;
            }
          }
        }
      }
      if (want_mask) {
        uint32_t wh = 0;
#pragma unroll
        for (int i = 0; i < K; i++) {
          const uint32_t rr = __reduce_or_sync(FULLMASK, lb[i]);
          wh |= ((rr >> lane) & 1u) << geo.bit(i);
          lb[i] = 0;
        }
        if (wh) atomicOr(&smask[gbase + lane], wh);
      }
      if (__all_sync(FULLMASK, done == ALL)) break;  // this warp's pixels are all saturated
    }
    bar.sync();  // everyone is done with this buffer before chunk c+2 is gathered into it; masks complete
    if (want_mask && tl < cnt) {
      strip_mask[range.x + (uint32_t)(c * NT + tl)] = (uint8_t)smask[tl];
      smask[tl] = 0;
    }
  }
  cp_async_wait<0>();

  const float bg0 = bg[0], bg1 = bg[1], bg2 = bg[2];
  const size_t HW = (size_t)H * W;
#pragma unroll
  for (int i = 0; i < K; i++) {
    const int y = pixy0 + 4 * i;
    if (pixx < W && y < H) {
      const size_t pix = (size_t)y * W + pixx;
      if (OUT & BLEND_OUT_FLOAT) {
        out_color[pix] = fmaf(T[i], bg0, Cr[i]);
        out_color[HW + pix] = fmaf(T[i], bg1, Cg[i]);
        out_color[2 * HW + pix] = fmaf(T[i], bg2, Cb[i]);
      }
      if (TRAIN && final_T != nullptr) {
        final_T[pix] = T[i];
        n_contrib[pix] = last[i];
      }
      if (DA) {
        if (out_alpha != nullptr) out_alpha[pix] = 1.0f - T[i];
        if (out_depth != nullptr) out_depth[pix] = D[i];
      }
    }
  }
  if (OUT & BLEND_OUT_U8) {
#pragma unroll
    for (int i = 0; i < K; i++)
      store_display<(OUT & BLEND_OUT_VIEWER) != 0>(out_rgb8, W, H, pixx, pixy0 + 4 * i, lane, fmaf(T[i], bg0, Cr[i]),
                                                   fmaf(T[i], bg1, Cg[i]), fmaf(T[i], bg2, Cb[i]));
  }
}

// CTA = 256 threads.  CTAs [0, n_heavy) take one heavy tile each on all eight warps; the following CTAs take four
// light tiles each, one per 64-thread group, K = 4.
// The view split and the training outputs are compile-time properties: either one at run time takes the plain forms
// from 64 registers (4 CTAs per SM) to 80 or more.  Occupancy bounds (DESIGN.md section 4): the plane forms
// GAB_FWD_DEPTH_CTAS, the K-view training form 3 (unbounded, ptxas holds it to 64 registers and spills); the plain
// forms are left to ptxas (minimum 0: no bound, which is not the same as 1).
template <int OUT, bool DA, bool VIEWS>
__global__ void __launch_bounds__(256, DA                                 ? GAB_FWD_DEPTH_CTAS
                                       : VIEWS && (OUT & BLEND_OUT_TRAIN) ? GAB_FWD_VIEWS_TRAIN_CTAS
                                                                          : 0) blend_forward_kernel(
    int W, int H, int gx, int tiles, int view_tiles, const uint2* __restrict__ ranges, const uint32_t* __restrict__ order,
    const uint32_t* __restrict__ order_info, const uint32_t* __restrict__ point_list, const SplatRec* __restrict__ rec,
    const float* __restrict__ bg, float* __restrict__ out_color, float* __restrict__ final_T,
    uint32_t* __restrict__ n_contrib, uint8_t* __restrict__ strip_mask, uint8_t* __restrict__ out_rgb8,
    float* __restrict__ out_alpha, float* __restrict__ out_depth) {
  __shared__ SplatRec buf[2][256];
  __shared__ uint32_t smask[256];
  __shared__ __align__(16) uint32_t ids_ring[4][ID_RING * (64 + 4)];  // per 64-thread group; a 256-thread tile uses it flat
  __shared__ __align__(8) uint64_t mbar[4][ID_RING];
  pdl_wait();
  pdl_trigger();
  const int nh = (int)order_info[0];
  const int b = blockIdx.x, t = threadIdx.x;
  if (b < nh) {
    forward_tile<1, OUT, DA, VIEWS>((int)order[b], t, GroupBarrier<256>{0}, buf[0], buf[1], smask, &ids_ring[0][0],
                                    mbar[0], W, H, gx, view_tiles, ranges, point_list, rec, bg, out_color, final_T,
                                    n_contrib, strip_mask, out_rgb8, out_alpha, out_depth);
  } else {
    const int g = t >> 6, slot = nh + 4 * (b - nh) + g;
    if (slot >= tiles) return;
    forward_tile<4, OUT, DA, VIEWS>((int)order[slot], t & 63, GroupBarrier<64>{1 + g}, buf[0] + g * 64,
                                    buf[1] + g * 64, smask + g * 64, ids_ring[g], mbar[g], W, H, gx, view_tiles, ranges,
                                    point_list, rec, bg, out_color, final_T, n_contrib, strip_mask, out_rgb8,
                                    out_alpha, out_depth);
  }
}

template <bool DA, bool VIEWS>
static decltype(&blend_forward_kernel<BLEND_OUT_FLOAT, DA, VIEWS>) blend_forward_instance(int out) {
  constexpr int F = BLEND_OUT_FLOAT, U = BLEND_OUT_U8, T = BLEND_OUT_TRAIN, V = BLEND_OUT_VIEWER;
  if constexpr (!DA) {  // the plane forms keep the training outputs at run time whatever OUT says
    if (out == (F | T)) return blend_forward_kernel<F | T, DA, VIEWS>;
    if (out == (F | U | T)) return blend_forward_kernel<F | U | T, DA, VIEWS>;
    // the viewer's quantisation: forward-only display forms without the planes (the entry points refuse the rest)
    if (out == (U | V)) return blend_forward_kernel<U | V, DA, VIEWS>;
    if (out == (F | U | V)) return blend_forward_kernel<F | U | V, DA, VIEWS>;
  }
  out &= F | U;
  return out == F ? blend_forward_kernel<F, DA, VIEWS>
         : out == U ? blend_forward_kernel<U, DA, VIEWS>
                    : blend_forward_kernel<F | U, DA, VIEWS>;
}

void launch_blend_forward(int views, int W, int H, const uint2* ranges, const uint32_t* order,
                          const uint32_t* order_info, const uint32_t* point_list, const SplatRec* rec, const float* bg,
                          float* out_color, float* final_T, uint32_t* n_contrib, uint8_t* strip_mask, uint8_t* out_rgb8,
                          float* out_alpha, float* out_depth, int quantize, cudaStream_t stream) {
  const int gx = (W + GAB_TILE - 1) / GAB_TILE, gy = (H + GAB_TILE - 1) / GAB_TILE;
  const int view_tiles = gx * gy, tiles = views * view_tiles;
  if (tiles == 0) return;
  const int out = (out_color != nullptr ? BLEND_OUT_FLOAT : 0) | (out_rgb8 != nullptr ? BLEND_OUT_U8 : 0) |
                  (final_T != nullptr ? BLEND_OUT_TRAIN : 0) |
                  (out_rgb8 != nullptr && quantize == GAB200_QUANTIZE_VIEWER ? BLEND_OUT_VIEWER : 0);
  const bool da = out_alpha != nullptr || out_depth != nullptr;
  auto kernel = da ? (views > 1 ? blend_forward_instance<true, true>(out) : blend_forward_instance<true, false>(out))
                   : (views > 1 ? blend_forward_instance<false, true>(out) : blend_forward_instance<false, false>(out));
  // upper bound on CTAs: every tile heavy; surplus CTAs exit at once
  launch_pdl(kernel, tiles, 256, 0, stream, W, H, gx, tiles, view_tiles, ranges, order, order_info, point_list, rec, bg,
             out_color, final_T, n_contrib, strip_mask, out_rgb8, out_alpha, out_depth);
}

// =====================================================================================================
// Backward
// =====================================================================================================
// Per-pixel state of the reverse walk (K pixels per lane, one per band).
// U is the dL/dpixel-weighted sum of everything behind the splat being visited, T_j included:
//   U_i = sum_{j>i} (c_j . d) alpha_j T_j + T_final (bg . d)        (d = dL/dpixel)
// so the reference's T_i ((c_i - colour behind) . d) - T_final (bg . d) / (1 - alpha_i) is T_i (c_i . d) - U_i / (1 -
// alpha_i), and one scalar per pixel replaces the three composited channels.
template <int K>
struct PixState {
  float fy[K];                // pixel row as float
  float T[K];                 // transmittance in front of the splat being visited (starts at final_T)
  float U[K];                 // sum behind the splat being visited (starts at final_T * (bg . dL/dpixel))
  float dr[K], dg[K], db[K];  // dL/dpixel
  int nc[K];                  // n_contrib: only list positions below it contributed to the pixel
};
struct SplatSums {  // per-lane sums over the lane's pixels for one splat; go = sum t, S1 = sum t dy, S2 = sum t dy^2
  float S1, S2, go, gr, gg, gb;  // with t = G dL/dalpha (dL/dG = opacity t: the opacity is applied once per visit)
};
// DA (depth plane): a fourth channel with colour z and background 0, z dL/ddepth in c . d, and alpha = 1 - T_final
// puts -T_final dL/dalpha into U's start
template <int K>
struct PixStateDA : PixState<K> {
  float dD[K];  // dL/ddepth
};
struct SplatSumsDA : SplatSums {
  float gz;     // dL/dz
};
template <int K, bool DA>
using PixStateT = std::conditional_t<DA, PixStateDA<K>, PixState<K>>;
template <bool DA>
using SplatSumsT = std::conditional_t<DA, SplatSumsDA, SplatSums>;

// One (splat, warp) visit restricted to the live bands M (compile-time set): straight-line code, the bands'
// dependency chains are independent and interleave.  A lane whose pixel did not receive this splat in the forward
// (beyond its n_contrib, outside the footprint, alpha < 1/255) runs the same instructions with alpha = G = 0 and
// T multiplied by exactly 1: every one of its contributions is an exact zero.
// FRESH: s holds nothing yet and the lowest band of M sets each sum instead of adding to it (no add of a zero).
template <int K, int M, bool DA = false, bool FRESH = false>
__device__ __forceinline__ void visit_bands(PixStateT<K, DA>& p, int pos, float py, float tA, float dx, float Bp,
                                            float Cp, float op, float cr, float cg, float cb, SplatSumsT<DA>& s,
                                            float cz = 0.f) {
#pragma unroll
  for (int i = 0; i < K; i++) {
    if (!((M >> i) & 1)) continue;
    const bool set = FRESH && (1 << i) == (M & -M);
    const float dy = py - p.fy[i];
    const float pw = fmaf(Cp * dy, dy, fmaf(Bp, dy, tA) * dx);  // the forward's expression, bit for bit
    const float G = ex2_approx(pw);
    const float alpha = fminf(0.99f, op * G);
    const bool valid = pos < p.nc[i] && pw <= 0.f && alpha >= ALPHA_MIN;
    const float al = valid ? alpha : 0.f;
    const float Gv = valid ? G : 0.f;
    const float ra = valid ? rcp_approx(1.f - alpha) : 1.f;
    const float Tn = p.T[i] * ra;  // transmittance in FRONT of this splat
    p.T[i] = Tn;
    const float w = al * Tn;
    s.gr = set ? w * p.dr[i] : fmaf(w, p.dr[i], s.gr);
    s.gg = set ? w * p.dg[i] : fmaf(w, p.dg[i], s.gg);
    s.gb = set ? w * p.db[i] : fmaf(w, p.db[i], s.gb);
    // dL/dalpha = T (c . dpix) - U / (1 - alpha)
    float cd = cr * p.dr[i];
    cd = fmaf(cg, p.dg[i], cd);
    cd = fmaf(cb, p.db[i], cd);
    if constexpr (DA) {
      cd = fmaf(cz, p.dD[i], cd);
      s.gz = set ? w * p.dD[i] : fmaf(w, p.dD[i], s.gz);
    }
    const float dLda = fmaf(Tn, cd, -p.U[i] * ra);
    p.U[i] = fmaf(w, cd, p.U[i]);  // the sum behind the NEXT (nearer) splat
    const float t = Gv * dLda;  // G dL/dalpha
    const float sd = t * dy;
    s.go = set ? t : s.go + t;
    s.S1 = set ? sd : s.S1 + sd;
    s.S2 = set ? sd * dy : fmaf(sd, dy, s.S2);
  }
}

// Dead bands skipped with warp-uniform branches, live bands one after the other (template recursion keeps the band
// index a compile-time constant, so p.X[i] stays in registers).
template <int K, int I, bool DA = false>
struct BandLoop {
  static __device__ __forceinline__ void run(uint32_t m, PixStateT<K, DA>& p, int pos, float py, float tA, float dx,
                                             float Bp, float Cp, float op, float cr, float cg, float cb,
                                             SplatSumsT<DA>& s, float cz = 0.f) {
    if (m & (1u << I)) visit_bands<K, (1 << I), DA>(p, pos, py, tA, dx, Bp, Cp, op, cr, cg, cb, s, cz);
    BandLoop<K, I + 1, DA>::run(m, p, pos, py, tA, dx, Bp, Cp, op, cr, cg, cb, s, cz);
  }
};
template <int K, bool DA>
struct BandLoop<K, K, DA> {
  static __device__ __forceinline__ void run(uint32_t, PixStateT<K, DA>&, int, float, float, float, float, float, float,
                                             float, float, float, SplatSumsT<DA>&, float = 0.f) {}
};

// Shared memory of one backward warp task: NR gradient components per splat (9; 10 with the depth plane's dL/dz).
// rows holds one batch of three visits, row slot * NR + component, one float per lane.  The stride of 36 floats puts
// the rows that eight consecutive lanes read with LDS.128 on eight different 4-bank groups (36 = 4 mod 32), so the
// lane-per-row loads are conflict-free; the stores (one row, 32 consecutive floats) are too.  One batch, not two: two
// padded batches (7.8 KB per warp, 8.6 KB with DA) would not let five 4-warp CTAs fit in the SM's 228 KB.
#define ROWS_STRIDE 36
template <int NR>
struct __align__(16) WarpSmemT {
  SplatRec rec[2][32];
  float rows[3 * NR][ROWS_STRIDE];  // [visit slot * NR + component][lane]
  uint32_t ids[ID_RING][32 + 4];
  uint8_t masks[ID_RING][32 + 16];
  uint64_t mbar[ID_RING];
};

// One warp task: the pixels of one (tile, half, band group), same ownership as the forward (BandGeom).
//   * The WARP is the unit of work.  It stages its own id/mask lists (TMA bulk copies into a private 3-slot ring) and
//     gathers only the records of entries that touch ITS blocks -- no CTA barrier anywhere, the warps of a tile drift
//     apart freely, and each walks only up to ITS pixels' largest n_contrib.
//   * A visit whose K bands are all live is one straight-line block, so the compiler interleaves the bands'
//     dependency chains; otherwise each band runs under a warp-uniform branch and dead bands cost nothing (BandLoop).
//   * The NR gradient components of three consecutive visits leave together through one BATCHED reduction: each
//     visit stores its NR per-lane values as rows slot * NR .. slot * NR + NR-1 of a shared-memory tile; after the
//     third, lane l < 3 NR loads row l (8 LDS.128), adds it with the same tree the single-visit reduction used (each
//     per-(warp, splat) sum is the same float) and issues the batch's one RED (27 lanes; 30 with DA); the walk's end
//     sends a partial batch.  The loads are not held across the next visit's band math: 32 more live floats there
//     spill at the 96-register bound of 5 CTAs per SM, so their latency is left to the SM's other warps.
// DA (gab200_backward_depth_alpha): records from the preprocess with DA (z in q2.w); dL_dalpha / dL_ddepth [H,W] or
// NULL (zero); a tenth component, dL/dz, leaves for g2d slot 9.
template <int K, bool DA>
__device__ __forceinline__ void backward_task(int tile, int tl, WarpSmemT<DA ? 10 : 9>& sm, int W, int H, int gx,
                                              const uint2* __restrict__ ranges,
                                              const uint32_t* __restrict__ point_list,
                                              const SplatRec* __restrict__ rec, const float* __restrict__ bg,
                                              const float* __restrict__ final_T,
                                              const uint32_t* __restrict__ n_contrib,
                                              const float* __restrict__ dL_dpix,
                                              const uint8_t* __restrict__ strip_mask, float* __restrict__ g2d,
                                              const float* __restrict__ dL_dalpha,
                                              const float* __restrict__ dL_ddepth) {
  constexpr int NR = DA ? 10 : 9;
  const int tx = tile % gx, ty = tile / gx;
  const int lane = tl & 31;
  const BandGeom<K> geo(tl);
  const int pixx = tx * GAB_TILE + geo.col;
  const int pixy0 = ty * GAB_TILE + geo.row0;
  const float fx = (float)pixx;
  const uint2 range = ranges[tile];
  const size_t HW = (size_t)H * W;
  const float bg0 = bg[0], bg1 = bg[1], bg2 = bg[2];

  PixStateT<K, DA> p;
  int n = 0;
#pragma unroll
  for (int i = 0; i < K; i++) {
    const int y = pixy0 + 4 * i;
    p.fy[i] = (float)y;
    float T0 = 0.f, dr = 0.f, dg = 0.f, db = 0.f, dA = 0.f, dZ = 0.f;
    p.nc[i] = 0;
    if (pixx < W && y < H) {
      const size_t pix = (size_t)y * W + pixx;
      T0 = final_T[pix];
      p.nc[i] = (int)n_contrib[pix];
      dr = dL_dpix[pix];
      dg = dL_dpix[HW + pix];
      db = dL_dpix[2 * HW + pix];
      if constexpr (DA) {
        if (dL_dalpha != nullptr) dA = dL_dalpha[pix];
        if (dL_ddepth != nullptr) dZ = dL_ddepth[pix];
      }
    }
    p.T[i] = T0;
    p.dr[i] = dr;
    p.dg[i] = dg;
    p.db[i] = db;
    if constexpr (DA) {  // alpha = 1 - T_final: dL/dT_final gains -dL/dalpha, which joins the background term
      p.U[i] = T0 * ((bg0 * dr + bg1 * dg + bg2 * db) - dA);
      p.dD[i] = dZ;
    } else {
      p.U[i] = T0 * (bg0 * dr + bg1 * dg + bg2 * db);
    }
    n = max(n, p.nc[i]);
  }
  // this warp only needs instances [0, max n_contrib of ITS pixels)
  n = __reduce_max_sync(FULLMASK, n);
  if (n == 0) return;
  const int nchunks = (n + 31) >> 5;
  const float half_W = 0.5f * (float)W, half_H = 0.5f * (float)H;

  constexpr uint32_t TX_BYTES = (32 + 4) * 4 + (32 + 16);
  auto chunk_lo = [&](int k) { return max(0, n - (k + 1) * 32); };
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < ID_RING; k++) mbar_init(&sm.mbar[k], 1);
    mbar_fence_init();
  }
  __syncwarp();
  auto issue_lists = [&](int k) {
    const uint32_t lo = range.x + (uint32_t)chunk_lo(k);
    uint64_t* b = &sm.mbar[k % ID_RING];
    mbar_arrive_expect_tx(b, TX_BYTES);
    bulk_copy_g2s(sm.ids[k % ID_RING], point_list + (lo & ~3u), (32 + 4) * 4, b);
    bulk_copy_g2s(sm.masks[k % ID_RING], strip_mask + (lo & ~15u), 32 + 16, b);
  };
  const int bit0 = geo.bit(0);
  // entry of chunk k owned by this lane: reverse index q = 32 k + lane <-> list position n-1-q
  auto stage_chunk = [&](int k, uint32_t& id, uint32_t& mine) {
    mbar_wait(&sm.mbar[k % ID_RING], (uint32_t)((k / ID_RING) & 1));
    const int q = k * 32 + lane;
    id = 0xffffffffu;
    mine = 0u;
    if (q < n) {
      const int lo = chunk_lo(k);
      const uint32_t g0 = range.x + (uint32_t)lo;
      const int rel = (n - 1 - q) - lo;
      id = sm.ids[k % ID_RING][(int)(g0 & 3u) + rel];
      const uint32_t mask = sm.masks[k % ID_RING][(int)(g0 & 15u) + rel];
#pragma unroll
      for (int i = 0; i < K; i++) mine |= ((mask >> (bit0 + 2 * i)) & 1u) << i;
      if (mine) gather_rec(&sm.rec[k & 1][lane], rec + id);
    }
    cp_async_commit();
  };
  if (lane == 0) {
    issue_lists(0);
    if (nchunks > 1) issue_lists(1);
  }
  uint32_t id_c, mine_c, id_n = 0xffffffffu, mine_n = 0u;
  stage_chunk(0, id_c, mine_c);

  // batch reduction state: `fill` visits (0..3, warp-uniform) have their rows in sm.rows; lane l < 3 NR owns row l,
  // component l % NR of the batch's visit l / NR, whose splat id is my_id.  Lanes >= 3 NR have my_slot = 3 and never
  // send anything.
  int fill = 0;
  const int my_slot = lane / NR;
  uint32_t my_id = 0xffffffffu;
  const float4* my_row = reinterpret_cast<const float4*>(sm.rows[min(lane, 3 * NR - 1)]);
  float* my_g2d = g2d + lane % NR;
  // the batch's rows -> g2d: lane l < 3 NR sums row l (8 LDS.128, the tree of the two 16-float halves, then their
  // sum) and sends it if a visit of this batch filled its slot
  auto send_batch = [&]() {
    __syncwarp();  // the rows of the batch's last visit are complete
    float h[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const float4 a = my_row[4 * k], b = my_row[4 * k + 1], c = my_row[4 * k + 2], d = my_row[4 * k + 3];
      h[k] = (((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w))) +
             (((c.x + c.y) + (c.z + c.w)) + ((d.x + d.y) + (d.z + d.w)));
    }
    if (my_slot < fill) atomicAdd(my_g2d + (size_t)my_id * GAB_G2D_STRIDE, h[0] + h[1]);
  };

  for (int c = 0; c < nchunks; c++) {
    __syncwarp();  // every lane is done with the record buffer and ring slot the next two lines overwrite
    if (c + 1 < nchunks) stage_chunk(c + 1, id_n, mine_n);  // its ids arrived while chunk c-1 was walked
    else cp_async_commit();
    if (lane == 0 && c + 2 < nchunks) issue_lists(c + 2);   // ring slot (c+2)%3 was last read for chunk c-1
    cp_async_wait<1>();
    __syncwarp();
    const SplatRec* cur = sm.rec[c & 1];
    uint32_t todo = __ballot_sync(FULLMASK, mine_c != 0u);
    while (todo) {
      const int jj = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t m = __shfl_sync(FULLMASK, mine_c, jj);
      const uint32_t id0 = __shfl_sync(FULLMASK, id_c, jj);
      const int pos = n - 1 - (c * 32 + jj);
      __syncwarp();  // a batch sent after the previous visit has been read; its slot 0 is free
      const float4 q0 = cur[jj].q0;
      const float4 q1 = cur[jj].q1;
      const float cbl = cur[jj].q2.x;
      const float czl = DA ? cur[jj].q2.w : 0.f;
      const float dx = q0.x - fx;
      const float tA = q0.z * dx;
      SplatSumsT<DA> s;
      if (m == (1u << K) - 1u) {
        visit_bands<K, (1 << K) - 1, DA, true>(p, pos, q0.y, tA, dx, q0.w, q1.x, q1.y, q1.z, q1.w, cbl, s, czl);
      } else {
        s.S1 = s.S2 = s.go = s.gr = s.gg = s.gb = 0.f;
        if constexpr (DA) s.gz = 0.f;
        BandLoop<K, 0, DA>::run(m, p, pos, q0.y, tA, dx, q0.w, q1.x, q1.y, q1.z, q1.w, cbl, s, czl);
      }
      const float A = q0.z * CONIC_UNSCALE_AC, B = q0.w * CONIC_UNSCALE_B, C = q1.x * CONIC_UNSCALE_AC;
      // sums of G dL/dG = opacity t
      const float S0 = q1.y * s.go, S1 = q1.y * s.S1, S2 = q1.y * s.S2;
      const float dxS0 = dx * S0;
      float* row = &sm.rows[fill * NR][lane];
      row[0 * ROWS_STRIDE] = (-A * dxS0 - B * S1) * half_W;  // dL/dmean2D.x (NDC units)
      row[1 * ROWS_STRIDE] = (-C * S1 - B * dxS0) * half_H;  // dL/dmean2D.y
      row[2 * ROWS_STRIDE] = -0.5f * dx * dxS0;              // dL/dconic.xx
      row[3 * ROWS_STRIDE] = -0.5f * dx * S1;                // dL/dconic.xy (stored once)
      row[4 * ROWS_STRIDE] = -0.5f * S2;                     // dL/dconic.yy
      row[5 * ROWS_STRIDE] = s.go;                             // dL/dopacity
      row[6 * ROWS_STRIDE] = s.gr;
      row[7 * ROWS_STRIDE] = s.gg;
      row[8 * ROWS_STRIDE] = s.gb;
      if constexpr (DA) row[9 * ROWS_STRIDE] = s.gz;         // dL/dz (view-space depth)
      if (my_slot == fill) my_id = id0;
      if (++fill == 3) {  // the batch is full
        send_batch();
        fill = 0;
      }
    }
    id_c = id_n;
    mine_c = mine_n;
  }
  cp_async_wait<0>();
  // the last, partial batch (a lane whose slot no visit of it filled sends nothing)
  if (fill > 0) send_batch();
}

// CTA = 128 threads: CTAs [0, n_heavy) take one heavy tile on four warps, K = 2; the rest take two light tiles each,
// two warps (the halves) per tile, K = 4.  5 CTAs per SM was the fastest occupancy measured on the H100.
// DA (gab200_backward*_depth_alpha): the alpha and depth plane gradients (backward_task<K, true>), either may be NULL
// (zero); bounded for GAB_BWD_DEPTH_CTAS CTAs per SM (DESIGN.md section 4 has the registers of both bounds).
// VIEWS (gab200_backward_views*): the K * view_tiles global tiles of a multi-view frame.  Global tile g is tile
// g % view_tiles of view g / view_tiles; its range, final_T, n_contrib and the pixel gradients are offset by view as
// the multi-view forward offsets them.  The point list holds virtual splat ids and the block masks are indexed by
// stream position, so records, masks and the K * P rows of g2d need no offset; backward_task runs unchanged.
template <bool DA, bool VIEWS>
__global__ void __launch_bounds__(128, DA ? GAB_BWD_DEPTH_CTAS : 5) blend_backward_kernel(
    int W, int H, int gx, int tiles, int view_tiles, const uint2* __restrict__ ranges,
    const uint32_t* __restrict__ order, const uint32_t* __restrict__ order_info, const uint32_t* __restrict__ point_list,
    const SplatRec* __restrict__ rec, const float* __restrict__ bg, const float* __restrict__ final_T,
    const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpix, const uint8_t* __restrict__ strip_mask,
    float* __restrict__ g2d, const float* __restrict__ dL_dalpha, const float* __restrict__ dL_ddepth) {
  __shared__ WarpSmemT<DA ? 10 : 9> sm[4];
  pdl_wait();
  pdl_trigger();
  const int nh = (int)order_info[1];
  const int b = blockIdx.x, t = threadIdx.x, w = t >> 5;
  const bool heavy = b < nh;
  const int slot = heavy ? b : nh + 2 * (b - nh) + (w >> 1);
  if (!heavy && slot >= tiles) return;
  const int tile = (int)order[slot];
  const int view = VIEWS ? tile / view_tiles : 0, local = tile - view * view_tiles;
  const size_t off = (size_t)view * H * W;
  const uint2* vr = ranges + (size_t)view * view_tiles;
  const float* va = dL_dalpha != nullptr ? dL_dalpha + off : nullptr;
  const float* vz = dL_ddepth != nullptr ? dL_ddepth + off : nullptr;
  if (heavy)  // heavy tile: four warps, two bands each
    backward_task<2, DA>(local, t, sm[w], W, H, gx, vr, point_list, rec, bg, final_T + off, n_contrib + off,
                         dL_dpix + 3 * off, strip_mask, g2d, va, vz);
  else        // two light tiles: two warps (the halves) each, four bands per warp
    backward_task<4, DA>(local, t & 63, sm[w], W, H, gx, vr, point_list, rec, bg, final_T + off, n_contrib + off,
                         dL_dpix + 3 * off, strip_mask, g2d, va, vz);
}

void launch_blend_backward(int views, int W, int H, const uint2* ranges, const uint32_t* order,
                           const uint32_t* order_info, const uint32_t* point_list, const SplatRec* rec, const float* bg,
                           const float* final_T, const uint32_t* n_contrib, const float* dL_dpix,
                           const uint8_t* strip_mask, float* g2d, bool da, const float* dL_dalpha,
                           const float* dL_ddepth, cudaStream_t stream) {
  const int gx = (W + GAB_TILE - 1) / GAB_TILE, gy = (H + GAB_TILE - 1) / GAB_TILE;
  const int view_tiles = gx * gy, tiles = views * view_tiles;
  if (tiles == 0) return;
  auto kernel = da ? (views > 1 ? blend_backward_kernel<true, true> : blend_backward_kernel<true, false>)
                   : (views > 1 ? blend_backward_kernel<false, true> : blend_backward_kernel<false, false>);
  launch_pdl(kernel, tiles, 128, 0, stream, W, H, gx, tiles, view_tiles, ranges, order, order_info, point_list, rec, bg,
             final_T, n_contrib, dL_dpix, strip_mask, g2d, dL_dalpha, dL_ddepth);
}

}  // namespace gab
