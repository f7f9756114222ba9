// tile_sort.cu -- the per-instance half of the tile|depth key sort as a COUNTING sort by tile + a per-tile sort by depth
// rank, as an alternative to cub::DeviceRadixSort over the instances (GAB200_TUNE_TILE_SORT = 1 selects it; cub is the
// default: every instance costs an atomic on its tile's counter in preprocess (RED) and another, with return value, in
// the emission, and the hot tiles (2000-3000 instances on one address) serialise the L2 atomic unit.  Kept because it
// needs no host-side N at all).
//
// The reference sorts N (tile << 32 | depth) keys with one LSD radix sort (SURVEY.md 2.4 K3-K5, Appendix B.2).  Stage A
// (binning.cu / preprocess.cu) already orders the SPLATS by (depth, id); a splat's position in that order -- its depth
// rank -- is a unique 32-bit key with exactly the reference's tie rule.  What remains is to group the instances by
// tile and order every tile's group by rank.  With the per-tile instance counts known before emission that needs no
// multi-pass sort over N:
//   preprocess_kernel      counts instances per tile while it computes each splat's tile spans (one RED per instance)
//   tile_scan_order_kernel exclusive scan of the counts -> ranges[tile] (what tile_ranges_kernel used to recover from
//                          key transitions), the per-tile write cursors, N, and the heaviest-first tile order
//   emit_keys_kernel       writes (rank, splat id) at cursor[tile]++ : each tile's segment is complete but unordered
//   tile_sort_kernel       one CTA per tile: ranks of the segment -> shared memory, bitonic sort (<= 2048 entries; one
//                          warp and no barrier for <= 32), ids written back in place
//   tile_sort_long_kernel  segments beyond 2048: a bitmap over all ranks in shared memory (ranks are unique) -- set one
//                          bit per entry, prefix-popcount, and the k-th set bit r lands at position k with id = order[r]
// 5 cub launches + 3 memsets + tile_ranges become 2 launches (3 when long tiles exist); the sorted stream is the
// reference's bit for bit (tests/test_gpu_parity.py, test_gpu_depth_sort.py run both implementations).
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

#define ORDER_NB 64
#define ORDER_WARPS 32
#define SCAN_NT 1024
#define ORDER_UNROLL 8

// Single CTA.  ranges / cursors from the per-tile counts, then the heaviest-first launch order of the tiles
// (longest-processing-time-first): the blend kernels walk one tile per CTA / warp pair and a tile's cost is
// proportional to its list length, so dispatching long lists first removes the tail where a few SMs grind through
// 2000-deep lists while the rest idle.  Counting sort into 64 length buckets; order_info[0/1] = number of tiles that
// are "heavy" for the forward / backward blend, order_info[2] = leading tiles of the order among which the ones longer
// than GAB_TILE_SORT_SMEM are (0 if there is none).
__global__ void __launch_bounds__(SCAN_NT) tile_scan_order_kernel(int tiles, const uint32_t* __restrict__ tile_count,
                                                                   uint32_t clamp, uint2* __restrict__ ranges,
                                                                   uint32_t* __restrict__ cursor,
                                                                   uint32_t* __restrict__ order,
                                                                   uint32_t* __restrict__ order_info,
                                                                   uint32_t* __restrict__ counters, int heavy_fwd,
                                                                   int heavy_bwd) {
  __shared__ uint32_t warp_tot[SCAN_NT / 32];
  __shared__ uint32_t s_carry;
  __shared__ uint32_t hist[ORDER_WARPS][ORDER_NB + 1];
  __shared__ uint32_t bucket_base[ORDER_NB];
  __shared__ uint32_t s_long;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  auto bucket = [](uint32_t len) -> int {
    return len == 0 ? ORDER_NB - 1 : (ORDER_NB - 2) - (int)min((uint32_t)(ORDER_NB - 2), len >> 5);
  };
  for (int k = tid; k < ORDER_WARPS * (ORDER_NB + 1); k += SCAN_NT) (&hist[0][0])[k] = 0;
  if (tid == 0) { s_carry = 0; s_long = 0; }
  __syncthreads();
  pdl_wait();  // shared-memory set-up above overlaps the predecessor; ranges / counts / order below
  pdl_trigger();
  if (tile_count != nullptr) {
    // ---- exclusive scan of the counts, SCAN_NT tiles per round ----
    for (int base = 0; base < tiles; base += SCAN_NT) {
      const int t = base + tid;
      const uint32_t c = t < tiles ? tile_count[t] : 0u;
      uint32_t incl = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += up;
      }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      uint32_t wbase = s_carry;
      for (int w = 0; w < warp; w++) wbase += warp_tot[w];
      const uint32_t start = wbase + incl - c;
      if (t < tiles) {
        // a frame that needs more than its capacity keeps what fits: [start, end) cut at `clamp` (emission drops the rest)
        ranges[t] = make_uint2(min(start, clamp), min(start + c, clamp));
        cursor[t] = start;
        atomicAdd(&hist[warp][bucket(min(start + c, clamp) - min(start, clamp))], 1u);
        if (c > GAB_TILE_SORT_SMEM) atomicAdd(&s_long, 1u);
      }
      __syncthreads();
      if (tid == SCAN_NT - 1) s_carry = wbase + incl;
      __syncthreads();
    }
    if (tid == 0) counters[GAB200_CTR_NUM_RENDERED] = s_carry;
  } else {
    // ranges were produced by tile_ranges_kernel (cub path): only the order is built here.  This CTA is alone on the
    // critical path between the sort and the blend: all of a thread's range loads are issued before the first
    // histogram update, so that the rounds do not pay one DRAM/L2 round trip each (8160 tiles = 8 rounds).
    for (int base = 0; base < tiles; base += ORDER_UNROLL * SCAN_NT) {
      uint32_t len[ORDER_UNROLL];
#pragma unroll
      for (int k = 0; k < ORDER_UNROLL; k++) {
        const int t = base + k * SCAN_NT + tid;
        len[k] = 0xffffffffu;
        if (t < tiles) {
          const uint2 r = ranges[t];
          len[k] = r.y - r.x;
        }
      }
#pragma unroll
      for (int k = 0; k < ORDER_UNROLL; k++)
        if (base + k * SCAN_NT + tid < tiles) atomicAdd(&hist[warp][bucket(len[k])], 1u);
    }
    __syncthreads();
  }
  // ---- bucket totals and per-warp starting offsets: thread b < ORDER_NB walks the warps of bucket b ----
  if (tid < ORDER_NB) {
    uint32_t run = 0;
    for (int w = 0; w < ORDER_WARPS; w++) {
      const uint32_t c = hist[w][tid];
      hist[w][tid] = run;  // exclusive offset of warp w inside the bucket
      run += c;
    }
    bucket_base[tid] = run;  // total
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t run = 0;
    // a tile is "heavy" for a pass when its list has >= heavy_* splats (multiples of 32): prefix of the order
    const int qf = min(ORDER_NB - 2, max(1, heavy_fwd >> 5)), qb = min(ORDER_NB - 2, max(1, heavy_bwd >> 5));
    for (int b = 0; b < ORDER_NB; b++) {
      const uint32_t c = bucket_base[b];
      bucket_base[b] = run;
      run += c;
      if (b == (ORDER_NB - 2) - qf) order_info[0] = run;
      if (b == (ORDER_NB - 2) - qb) order_info[1] = run;
      // bucket 0 holds every list of 1984 entries or more, in no particular order: when any of them is beyond the
      // shared-memory sort, tile_sort_long_kernel looks at all of bucket 0 (and skips the ones that are not)
      if (b == 0) order_info[2] = s_long ? c : 0u;
    }
  }
  __syncthreads();
  // warp w of round r sees the same tiles as in the counting loop above (same t -> same warp), so its private
  // cursor row hist[w][*] hands out exactly the slots it counted
  for (int base = 0; base < tiles; base += ORDER_UNROLL * SCAN_NT) {
    uint32_t len[ORDER_UNROLL];
#pragma unroll
    for (int k = 0; k < ORDER_UNROLL; k++) {
      const int t = base + k * SCAN_NT + tid;
      len[k] = 0u;
      if (t < tiles) {
        const uint2 r = ranges[t];
        len[k] = r.y - r.x;
      }
    }
#pragma unroll
    for (int k = 0; k < ORDER_UNROLL; k++) {
      const int t = base + k * SCAN_NT + tid;
      if (t < tiles) {
        const int b = bucket(len[k]);
        order[bucket_base[b] + atomicAdd(&hist[warp][b], 1u)] = (uint32_t)t;
      }
    }
  }
}

void launch_tile_scan_order(int tiles, const uint32_t* tile_count, uint32_t clamp, uint2* ranges, uint32_t* cursor,
                            uint32_t* order, uint32_t* order_info, uint32_t* counters, int heavy_fwd, int heavy_bwd,
                            cudaStream_t stream) {
  if (tiles == 0) return;
  launch_pdl(tile_scan_order_kernel, 1, SCAN_NT, 0, stream, tiles, tile_count, clamp, ranges, cursor, order, order_info,
             counters, heavy_fwd, heavy_bwd);
}

// =====================================================================================================
// per-tile sort by depth rank
// =====================================================================================================
#define TS_NT 128
__global__ void __launch_bounds__(TS_NT) tile_sort_kernel(int tiles, const uint2* __restrict__ ranges,
                                                          const uint32_t* __restrict__ order,
                                                          uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  __shared__ uint32_t sk[GAB_TILE_SORT_SMEM];
  __shared__ uint32_t sv[GAB_TILE_SORT_SMEM];
  const int tile = (int)order[blockIdx.x];
  const uint2 r = ranges[tile];
  const int n = (int)(r.y - r.x);
  if (n <= 1 || n > GAB_TILE_SORT_SMEM) return;  // long segments: tile_sort_long_kernel
  const int tid = threadIdx.x;
  uint32_t* k = keys + r.x;
  uint32_t* v = vals + r.x;
  if (n <= 32) {
    // one warp, no shared memory: rank of every entry = number of smaller keys (keys are distinct)
    if (tid >= 32) return;
    const uint32_t key = tid < n ? k[tid] : 0xffffffffu;
    const uint32_t val = tid < n ? v[tid] : 0u;
    int rank = 0;
#pragma unroll 8
    for (int j = 0; j < 32; j++) rank += __shfl_sync(0xffffffffu, key, j) < key ? 1 : 0;
    if (tid < n) v[rank] = val;  // every lane has loaded its input: in-place scatter is safe after the shuffles
    return;
  }
  int m = 64;
  while (m < n) m <<= 1;
  for (int i = tid; i < m; i += TS_NT) {
    sk[i] = i < n ? k[i] : 0xffffffffu;
    sv[i] = i < n ? v[i] : 0u;
  }
  __syncthreads();
  for (int size = 2; size <= m; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < (m >> 1); t += TS_NT) {
        const int lo = 2 * t - (t & (stride - 1));  // index with bit `stride` clear
        const int hi = lo + stride;
        const bool up = (lo & size) == 0;
        const uint32_t a = sk[lo], b = sk[hi];
        if ((a > b) == up) {
          sk[lo] = b; sk[hi] = a;
          const uint32_t x = sv[lo]; sv[lo] = sv[hi]; sv[hi] = x;
        }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < n; i += TS_NT) v[i] = sv[i];
}

// Segments longer than the shared-memory sort: ranks are unique integers below `listed`, so a tile's sorted list is
// the ascending enumeration of a bitmap.  `words_cap` bits-words of dynamic shared memory cover the ranks in passes.
#define TSL_NT 1024
__global__ void __launch_bounds__(TSL_NT) tile_sort_long_kernel(const uint2* __restrict__ ranges,
                                                                const uint32_t* __restrict__ order,
                                                                const uint32_t* __restrict__ order_info,
                                                                const uint32_t* __restrict__ keys,
                                                                uint32_t* __restrict__ vals,
                                                                const uint32_t* __restrict__ rank_to_id,
                                                                const uint32_t* __restrict__ listed_ptr, int P,
                                                                int words_cap) {
  extern __shared__ uint32_t bits[];
  __shared__ uint32_t warp_tot[TSL_NT / 32];
  __shared__ uint32_t s_base;
  const int nlong = (int)order_info[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t listed = listed_ptr != nullptr ? min(*listed_ptr, (uint32_t)P) : (uint32_t)P;
  const int total_words = (int)((listed + 31u) >> 5);
  // the long tiles are among the first `nlong` of the heaviest-first order
  for (int slot = blockIdx.x; slot < nlong; slot += gridDim.x) {
    const int tile = (int)order[slot];
    const uint2 r = ranges[tile];
    const int n = (int)(r.y - r.x);
    if (n <= GAB_TILE_SORT_SMEM) continue;
    if (tid == 0) s_base = 0;
    for (int w0 = 0; w0 < total_words; w0 += words_cap) {  // one pass per window of ranks
      const int nw = min(words_cap, total_words - w0);
      for (int i = tid; i < nw; i += TSL_NT) bits[i] = 0;
      __syncthreads();
      const uint32_t lo = (uint32_t)w0 << 5, hi = (uint32_t)(w0 + nw) << 5;
      for (int i = tid; i < n; i += TSL_NT) {
        const uint32_t rk = keys[r.x + i];
        if (rk >= lo && rk < hi) atomicOr(&bits[(rk - lo) >> 5], 1u << (rk & 31u));
      }
      __syncthreads();
      // enumerate the set bits in ascending order: thread t owns a contiguous run of words
      const int per = (nw + TSL_NT - 1) / TSL_NT;
      const int a = min(tid * per, nw), b = min(a + per, nw);
      uint32_t cnt = 0;
      for (int i = a; i < b; i++) cnt += __popc(bits[i]);
      uint32_t incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += up;
      }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      uint32_t pos = s_base + incl - cnt;
      for (int w = 0; w < warp; w++) pos += warp_tot[w];
      for (int i = a; i < b; i++) {
        uint32_t word = bits[i];
        while (word) {
          const int bit = __ffs(word) - 1;
          word &= word - 1;
          vals[r.x + pos++] = rank_to_id[lo + ((uint32_t)i << 5) + (uint32_t)bit];
        }
      }
      __syncthreads();
      if (tid == TSL_NT - 1) s_base = pos;  // the last thread's end = total so far (its run is the last one)
      __syncthreads();
    }
  }
}

void launch_tile_sort(int tiles, const uint2* ranges, const uint32_t* order, const uint32_t* order_info, uint32_t* keys,
                      uint32_t* vals, const uint32_t* rank_to_id, const uint32_t* listed, int P, cudaStream_t stream) {
  if (tiles == 0) return;
  tile_sort_kernel<<<tiles, TS_NT, 0, stream>>>(tiles, ranges, order, keys, vals);
  count_launch();
  // long tiles (none at the headline sizes; order_info[2] is only known on the device, so the kernel is always
  // enqueued and exits at once when there is nothing to do)
  static int smem_words = 0;
  if (smem_words == 0) {
    int dev = 0, max_optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    int bytes = max_optin - 1024;  // static arrays of the kernel
    if (bytes > 160 * 1024) bytes = 160 * 1024;
    if (bytes < 32 * 1024) bytes = 32 * 1024;
    cudaFuncSetAttribute(tile_sort_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    smem_words = bytes / 4;
  }
  int need_words = (P + 31) / 32;
  if (need_words > smem_words) need_words = smem_words;
  if (need_words < 1) need_words = 1;
  tile_sort_long_kernel<<<GAB_NUM_SMS, TSL_NT, (size_t)need_words * 4, stream>>>(ranges, order, order_info, keys, vals,
                                                                         rank_to_id, listed, P, need_words);
  count_launch();
}

// the reference's key format (tile << 32 | fp32 depth bits) rebuilt from the ranges (parity export)
__global__ void expand_keys_by_range_kernel(int tiles, const uint2* __restrict__ ranges, const uint32_t* __restrict__ ids,
                                            const SplatAux* __restrict__ aux, uint64_t* __restrict__ out) {
  const int tile = blockIdx.x;
  const uint2 r = ranges[tile];
  for (uint32_t i = r.x + threadIdx.x; i < r.y; i += blockDim.x)
    out[i] = ((uint64_t)tile << 32) | (uint64_t)__float_as_uint(aux[ids[i]].depth);
}
void launch_expand_keys_by_range(int tiles, const uint2* ranges, const uint32_t* ids, const SplatAux* aux, uint64_t* out,
                                 cudaStream_t stream) {
  if (tiles == 0) return;
  expand_keys_by_range_kernel<<<tiles, 128, 0, stream>>>(tiles, ranges, ids, aux, out);
  count_launch();
}

}  // namespace gab
