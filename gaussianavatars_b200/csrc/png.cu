// png.cu -- PNG files written on the device (gab200_png_bound / gab200_png_scratch_bytes / gab200_png_encode /
// gab200_png_copy): 8-bit RGB, not interlaced, chunks signature | IHDR | one IDAT | IEND, the IDAT data one zlib stream.
//
// Per view the encode runs six kernels, each named for a trace:
//   png_filter_kernel   one CTA per row: the five PNG filters, the one with the least sum of |signed byte| (ties: the
//                       lowest filter id, libpng's heuristic; oracle/png.py restates it) -> the filtered stream
//                       (H rows of 1 + 3W bytes).  It also zeroes the view's deflate buffer.
//   png_lz_kernel       one 1024-thread CTA per segment: PNG_SEG bytes of the filtered stream (the last one shorter),
//                       staged in shared memory with the PNG_WIN bytes before it (matches reach back into earlier
//                       segments of the same view, never into another view).  Per position the longest match of five
//                       candidates -- distance 1, 3 (the previous pixel), the nearest position of the same 3-byte hash
//                       up to 256 back in the position's round of 1024, 3W + 1 (the previous row, when <= 32768) and
//                       the latest position of the same hash before the round (a table refreshed every 1024
//                       positions) -- ties to the earlier candidate in that order.  The greedy parse (next = p +
//                       max(1, len)) is walked by pointer doubling: 15 rounds mark every position the parse from the
//                       segment's first byte reaches.  Then the segment's dynamic Huffman codes (literal/length limited to 15 bits,
//                       code-length codes to 7, the RLE codes 16/17/18 in the header; deterministic: leaves ordered by
//                       (count, symbol)), the exact bit cost of the dynamic and the fixed block, and the smaller of the
//                       two (ties: fixed) rendered at bit 0 of the segment's staging area, unless even a stored block
//                       would be smaller.  The segment's Adler-32 goes beside it.
//   png_offsets_kernel  one thread per view walks the segments in order: the exact stored cost at the bit offset the
//                       segment starts at (a stored block pads to a byte), the block kind (the smallest; ties: stored,
//                       then the Huffman block), the segment's bit offset, the view's Adler-32 (adler32_combine) and
//                       the file length, written to out_len[view].
//   png_pack_kernel     one CTA per segment: its bits at their offset in the deflate buffer; the first and last word
//                       of a segment are OR-ed in with atomics (a neighbour shares them), so the result does not
//                       depend on the order the CTAs run in.  The last block gets BFINAL.
//   png_assemble_kernel one CTA per 64 KiB of the IDAT chunk: the zlib header 78 01, the deflate bytes and the
//                       Adler-32 into the file, and the piece's CRC-32 (per-thread CRCs of contiguous runs, combined as
//                       zlib's crc32_combine does).
//   png_finish_kernel   one CTA per view: the pieces' CRCs combined in order; signature, IHDR, the IDAT's length and
//                       CRC-32, IEND.
// No file exceeds gab200_png_bound(W, H) = 63 + n + 6 S (n = H (3W + 1) filtered bytes, S = ceil(n / PNG_SEG)): every
// block is at most its stored form, 42 bits of header and padding plus its bytes.
#include "common.cuh"
#include "deflate.cuh"
#include "kernels.cuh"

namespace gab {

namespace {

constexpr int PNG_SEG = 32768;         // filtered bytes per segment (one deflate block)
constexpr int PNG_WIN = 32768;         // the deflate window
constexpr int LZ_THREADS = 1024;
constexpr int PER_THREAD = PNG_SEG / LZ_THREADS;   // 32
constexpr int HASH_BITS = 13;
constexpr int HASH_SIZE = 1 << HASH_BITS;
constexpr int MAX_MATCH = 258;
constexpr int NEAR_SCAN = 256;         // positions of the current round searched back for the same 3-byte hash
constexpr int LIT_SYMS = 286, DIST_SYMS = 30, CL_SYMS = 19;
constexpr uint32_t NO_HUFF = 0xffffffffu;
// staging words per segment: the largest Huffman block ever rendered is the stored bound of a whole segment
constexpr int STAGE_WORDS = (42 + 8 * PNG_SEG + 31) / 32 + 2;
// dynamic shared memory of png_lz_kernel: the bytes (then the parse's jump table, then the rendered bits), one record
// per position, the hash table (then the Huffman tables)
constexpr int LZ_BUF_BYTES = PNG_WIN + PNG_SEG;
constexpr int LZ_SMEM = LZ_BUF_BYTES + 4 * PNG_SEG + 4 * HASH_SIZE;
constexpr unsigned FULL = 0xffffffffu;
constexpr int ASM_CHUNK = 65536;       // bytes of the IDAT chunk per png_assemble_kernel CTA

// record of a position (rec[]): bit 31 the parse reaches it; len = bits 0..8 (0: a literal, byte in bits 9..16; else
// 3..258 with the distance - 1 in bits 9..23)
constexpr uint32_t MARK = 0x80000000u;

struct SegMeta {
  uint32_t huff_bits;   // bits of the rendered Huffman block, NO_HUFF when none was rendered
  uint32_t n;           // filtered bytes of the segment
  uint32_t adler;       // Adler-32 of those bytes
  uint32_t stored;      // set by png_offsets_kernel: 1 = a stored block
  int64_t off;          // set by png_offsets_kernel: the block's first bit in the deflate stream
  int64_t pad;
};
static_assert(sizeof(SegMeta) == 32, "SegMeta is 32 bytes");

struct ViewMeta {
  int64_t total_bits;   // bits of the deflate stream
  uint32_t adler;
  uint32_t idat_len;    // IDAT data bytes: zlib header, deflate bytes, Adler-32
};

__host__ __device__ inline int64_t filtered_bytes(int H, int W) { return (int64_t)H * (3 * (int64_t)W + 1); }
__host__ __device__ inline int64_t segments_of(int64_t n) { return (n + PNG_SEG - 1) / PNG_SEG; }
__host__ __device__ inline int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }
// words of the deflate buffer of one view: the stored bound of the stream, plus a word of slack
__host__ __device__ inline int64_t deflate_words(int64_t n) { return round_up((n + 6 * segments_of(n)) / 4 + 2, 64); }

struct Layout {
  uint8_t* filt;      // [views][filt_stride]
  uint32_t* defl;     // [views][defl_words]
  uint32_t* stage;    // [views * S][STAGE_WORDS]
  SegMeta* seg;       // [views * S]
  ViewMeta* view;     // [views]
  uint2* crc;         // [views][chunks]: CRC-32 and length of each ASM_CHUNK piece of the IDAT chunk
  int64_t filt_stride, defl_words, S, chunks;
  size_t bytes;       // the scratch the layout takes
};

__host__ __device__ inline Layout carve(void* scratch, int64_t views, int H, int W) {
  Layout l;
  const int64_t n = filtered_bytes(H, W);
  l.S = segments_of(n);
  l.filt_stride = round_up(n, 256);
  l.defl_words = deflate_words(n);
  Carver c(scratch);
  l.filt = c.take<uint8_t>(views * l.filt_stride);
  l.defl = c.take<uint32_t>(views * l.defl_words);
  l.stage = c.take<uint32_t>(views * l.S * STAGE_WORDS);
  l.seg = c.take<SegMeta>(views * l.S);
  l.view = c.take<ViewMeta>(views);
  l.chunks = (4 + 6 + n + 6 * l.S + ASM_CHUNK - 1) / ASM_CHUNK;   // the IDAT's type and largest data
  l.crc = c.take<uint2>(views * l.chunks);
  l.bytes = c.bytes();
  return l;
}

// ---- checksums ----------------------------------------------------------------------------------------------------
constexpr uint32_t CRC_POLY = 0xedb88320u;

// a * b modulo the CRC-32 polynomial (reflected), as zlib's multmodp
__device__ uint32_t crc_multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}

// zlib's crc32_combine: the CRC-32 of A || B from those of A and B and B's length (x2n[k] = x^(2^k) mod P)
__device__ uint32_t crc_combine(uint32_t c1, uint32_t c2, uint64_t len2, const uint32_t* x2n) {
  uint32_t p = 1u << 31;   // x^0
  int k = 3;               // x^(8 len2)
  while (len2) {
    if (len2 & 1) p = crc_multmodp(x2n[k & 31], p);
    len2 >>= 1;
    k++;
  }
  return crc_multmodp(p, c1) ^ c2;
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24);
  p[1] = (uint8_t)(v >> 16);
  p[2] = (uint8_t)(v >> 8);
  p[3] = (uint8_t)v;
}

// ---- block-wide helpers (LZ_THREADS threads) ----------------------------------------------------------------------
// exclusive scan of one uint32 per thread; *total gets the sum.  red: 32 words of shared memory.
__device__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* red, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(FULL, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) red[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = red[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(FULL, w, o);
      if (lane >= o) w += y;
    }
    red[lane] = w;
  }
  __syncthreads();
  const uint32_t before = (warp > 0 ? red[warp - 1] : 0u) + x - v;
  *total = red[31];
  __syncthreads();
  return before;
}

// ---- deflate symbol tables ------------------------------------------------------------------------------------------
__device__ __forceinline__ void length_code(int len, int& sym, int& ebits, int& eval) {
  if (len == 258) {
    sym = 285, ebits = 0, eval = 0;
    return;
  }
  const int x = len - 3;
  if (x < 8) {
    sym = 257 + x, ebits = 0, eval = 0;
    return;
  }
  const int n = 31 - __clz(x);
  sym = 257 + 4 * (n - 1) + ((x >> (n - 2)) & 3);
  ebits = n - 2;
  eval = x & ((1 << (n - 2)) - 1);
}

__device__ __forceinline__ void dist_code(int dist, int& sym, int& ebits, int& eval) {
  const int x = dist - 1;
  if (x < 4) {
    sym = x, ebits = 0, eval = 0;
    return;
  }
  const int n = 31 - __clz(x);
  sym = 2 * n + ((x >> (n - 1)) & 1);
  ebits = n - 1;
  eval = x & ((1 << (n - 1)) - 1);
}

__device__ __forceinline__ int fixed_lit_len(int s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }

__device__ __forceinline__ uint32_t bit_reverse(uint32_t code, int len) { return __brev(code) >> (32 - len); }

// Code lengths of n symbols with counts freq[] (m >= 2 of them nonzero, listed in order[] by (count, symbol)), limited
// to maxbits: Moffat and Katajainen's in-place minimum-redundancy lengths, then the length limit as miniz enforces it
// (the deepest leaves move up until the Kraft sum is exact), the longest codes to the rarest leaves.  One thread.
// work[]: m entries of scratch; len[] gets the lengths (0 for an unused symbol).
__device__ void huffman_lengths(const uint32_t* freq, int n, int m, int maxbits, const uint16_t* order, uint32_t* work,
                                uint8_t* len) {
  for (int s = 0; s < n; s++) len[s] = 0;
  for (int i = 0; i < m; i++) work[i] = freq[order[i]];
  // first pass: parent pointers
  uint32_t* A = work;
  A[0] += A[1];
  int root = 0, leaf = 2;
  for (int next = 1; next < m - 1; next++) {
    if (leaf >= m || A[root] < A[leaf]) {
      A[next] = A[root];
      A[root++] = next;
    } else {
      A[next] = A[leaf++];
    }
    if (leaf >= m || (root < next && A[root] < A[leaf])) {
      A[next] += A[root];
      A[root++] = next;
    } else {
      A[next] += A[leaf++];
    }
  }
  // second pass: internal depths; third pass: leaf depths
  A[m - 2] = 0;
  for (int next = m - 3; next >= 0; next--) A[next] = A[A[next]] + 1;
  int avbl = 1, used = 0, dpth = 0;
  root = m - 2;
  int next = m - 1;
  while (avbl > 0) {
    while (root >= 0 && (int)A[root] == dpth) {
      used++;
      root--;
    }
    while (avbl > used) {
      A[next--] = dpth;
      avbl--;
    }
    avbl = 2 * used;
    dpth++;
    used = 0;
  }
  // A[i]: the depth of leaf order[i] (non-increasing in i).  Count per length, fold anything deeper than maxbits.
  int count[33];
  for (int i = 0; i <= 32; i++) count[i] = 0;
  for (int i = 0; i < m; i++) count[min((int)A[i], 32)]++;
  for (int i = maxbits + 1; i <= 32; i++) {
    count[maxbits] += count[i];
    count[i] = 0;
  }
  uint32_t total = 0;
  for (int i = maxbits; i > 0; i--) total += (uint32_t)count[i] << (maxbits - i);
  while (total != (1u << maxbits)) {
    count[maxbits]--;
    for (int i = maxbits - 1; i > 0; i--) {
      if (count[i]) {
        count[i]--;
        count[i + 1] += 2;
        break;
      }
    }
    total--;
  }
  int j = m;
  for (int l = 1; l <= maxbits; l++)
    for (int c = count[l]; c > 0; c--) len[order[--j]] = (uint8_t)l;
}

// canonical codes of lengths len[0..n), bit-reversed for LSB-first packing: code | length << 16
__device__ void canonical_codes(const uint8_t* len, int n, uint32_t* code) {
  int count[16], next[16];
  for (int i = 0; i < 16; i++) count[i] = 0;
  for (int s = 0; s < n; s++) count[len[s]]++;
  count[0] = 0;
  int c = 0;
  for (int b = 1; b < 16; b++) {
    c = (c + count[b - 1]) << 1;
    next[b] = c;
  }
  for (int s = 0; s < n; s++) {
    const int l = len[s];
    code[s] = l ? bit_reverse((uint32_t)next[l]++, l) | ((uint32_t)l << 16) : 0u;
  }
}

// at least two used symbols in every tree (zlib's rule: an inflater accepts no incomplete code): the lowest unused
// symbols get a count of one; they cost header bits only
__device__ void two_used(uint32_t* freq, int n) {
  int used = 0;
  for (int s = 0; s < n; s++) used += freq[s] != 0;
  for (int s = 0; s < n && used < 2; s++)
    if (freq[s] == 0) {
      freq[s] = 1;
      used++;
    }
}

// OR `nbits` (<= 57) bits of v at bit `off` of the word stream w (shared memory)
__device__ __forceinline__ void put_bits(uint32_t* w, uint32_t off, uint64_t v, int nbits) {
  if (nbits == 0) return;
  const uint32_t i = off >> 5, s = off & 31;
  const uint64_t lo = v << s;   // bits s .. s + nbits - 1 (< 64 when s + nbits <= 64)
  atomicOr(w + i, (uint32_t)lo);
  if (s + nbits > 32) atomicOr(w + i + 1, (uint32_t)(lo >> 32));
  if (s + nbits > 64) atomicOr(w + i + 2, (uint32_t)(v >> (64 - s)));
}

// The Huffman tables of one segment (shared memory, in the hash table's space once the matches are found)
struct HuffSmem {
  uint32_t lit_freq[LIT_SYMS];
  uint32_t dist_freq[DIST_SYMS];
  uint32_t cl_freq[CL_SYMS];
  uint32_t lit_code[LIT_SYMS];    // bit-reversed code | length << 16, of the block being rendered
  uint32_t dist_code[DIST_SYMS];
  uint32_t cl_code[CL_SYMS];
  uint8_t lit_len[LIT_SYMS];
  uint8_t dist_len[DIST_SYMS];
  uint8_t cl_len[CL_SYMS];
  uint8_t pad0;
  uint16_t rle[LIT_SYMS + DIST_SYMS];   // code-length symbol | extra value << 5
  uint16_t order_a[LIT_SYMS];
  uint16_t order_b[DIST_SYMS + 2];
  uint32_t work_a[LIT_SYMS];
  uint32_t work_b[DIST_SYMS + 2];
  uint32_t n_rle, hlit, hdist, hclen, header_bits;
  uint32_t extra_bits;                  // the length and distance extra bits of the segment's matches
  uint32_t use_fixed, huff_bits;
};
static_assert(sizeof(HuffSmem) <= 4 * HASH_SIZE, "the Huffman tables live in the hash table's space");

__device__ __forceinline__ uint32_t load4(const uint32_t* w, uint32_t off) {
  return __funnelshift_r(w[off >> 2], w[(off >> 2) + 1], 8 * (off & 3));
}

// the match length (0 if < 3) of the bytes at `at` against those `dist` before, at most `maxlen`
__device__ __forceinline__ int match_len(const uint8_t* buf, const uint32_t* buf32, uint32_t at, uint32_t dist,
                                         int maxlen) {
  const uint32_t src = at - dist;
  int l = 0;
  while (l + 4 <= maxlen) {
    const uint32_t x = load4(buf32, at + l) ^ load4(buf32, src + l);
    if (x) return l + ((__ffs(x) - 1) >> 3);
    l += 4;
  }
  while (l < maxlen && buf[at + l] == buf[src + l]) l++;
  return l;
}

// The shortest match worth its distance: a far match's distance code and extra bits cost more than three or four
// literals of a rendered image's filtered residuals
__device__ __forceinline__ int min_match(uint32_t dist) { return dist <= 64 ? 3 : dist <= 4096 ? 4 : 5; }

__device__ __forceinline__ uint32_t hash3(const uint8_t* buf, uint32_t at) {
  const uint32_t v = (uint32_t)buf[at] | ((uint32_t)buf[at + 1] << 8) | ((uint32_t)buf[at + 2] << 16);
  return (v * 2654435761u) >> (32 - HASH_BITS);
}

// ---- kernels ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) png_filter_kernel(int H, int W, const uint8_t* __restrict__ rgb, Layout l) {
  const int y = blockIdx.x, k = blockIdx.y;
  const int64_t rowb = 3 * (int64_t)W;
  const uint8_t* cur = rgb + ((int64_t)k * H + y) * rowb;
  const uint8_t* prev = y > 0 ? cur - rowb : nullptr;
  // this row's share of zeroing the view's deflate buffer
  {
    uint32_t* d = l.defl + k * l.defl_words;
    const int64_t per = (l.defl_words + H - 1) / H, a = (int64_t)y * per, b = min(a + per, l.defl_words);
    for (int64_t i = a + threadIdx.x; i < b; i += blockDim.x) d[i] = 0;
  }
  auto filt = [&](int f, int64_t x) -> uint8_t {
    const int r = cur[x];
    const int a = x >= 3 ? cur[x - 3] : 0, b = prev ? prev[x] : 0, c = (prev && x >= 3) ? prev[x - 3] : 0;
    int pred = 0;
    if (f == 1) pred = a;
    else if (f == 2) pred = b;
    else if (f == 3) pred = (a + b) >> 1;
    else if (f == 4) {
      const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
      pred = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
    }
    return (uint8_t)(r - pred);
  };
  uint32_t sum[5] = {0, 0, 0, 0, 0};
  for (int64_t x = threadIdx.x; x < rowb; x += blockDim.x) {
#pragma unroll
    for (int f = 0; f < 5; f++) {
      const uint32_t v = filt(f, x);
      sum[f] += v < 128 ? v : 256 - v;
    }
  }
  __shared__ uint32_t red[8][5];
  __shared__ int chosen;
#pragma unroll
  for (int f = 0; f < 5; f++) {
    uint32_t v = sum[f];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(FULL, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][f] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    uint32_t bs = 0;
    for (int f = 0; f < 5; f++) {
      uint32_t s = 0;
      for (int w = 0; w < 8; w++) s += red[w][f];
      if (f == 0 || s < bs) best = f, bs = s;   // ties: the lowest filter id
    }
    chosen = best;
  }
  __syncthreads();
  const int f = chosen;
  uint8_t* out = l.filt + k * l.filt_stride + (int64_t)y * (rowb + 1);
  if (threadIdx.x == 0) out[0] = (uint8_t)f;
  for (int64_t x = threadIdx.x; x < rowb; x += blockDim.x) out[1 + x] = filt(f, x);
}

__global__ void __launch_bounds__(LZ_THREADS, 1) png_lz_kernel(int W, int64_t n_total, Layout l) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* buf = smem;                                               // window + segment bytes
  uint32_t* buf32 = reinterpret_cast<uint32_t*>(smem);
  uint32_t* rec = reinterpret_cast<uint32_t*>(smem + LZ_BUF_BYTES);  // one record per segment position
  uint32_t* hash = rec + PNG_SEG;
  HuffSmem& hs = *reinterpret_cast<HuffSmem*>(hash);
  uint16_t* jump = reinterpret_cast<uint16_t*>(smem);                // the parse's jump table, in buf's space
  uint32_t* bits = buf32;                                            // the rendered block, in buf's space
  __shared__ uint32_t red[32];
  __shared__ uint32_t red2[32];
  __shared__ uint16_t round_hash[LZ_THREADS];

  const int s = blockIdx.x, k = blockIdx.y, t = threadIdx.x;
  const int64_t start = (int64_t)s * PNG_SEG;
  const int n_seg = (int)min((int64_t)PNG_SEG, n_total - start);
  const int64_t ws = max((int64_t)0, start - PNG_WIN);
  const int n_win = (int)(start - ws);
  const int n_buf = n_win + n_seg;
  const uint8_t* src = l.filt + k * l.filt_stride + ws;   // 16-byte aligned: ws is a multiple of PNG_SEG
  SegMeta& meta = l.seg[(int64_t)k * l.S + s];

  // stage the bytes; zero the hash table
  for (int i = t; i < n_buf / 16; i += LZ_THREADS)
    reinterpret_cast<uint4*>(buf)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
  for (int i = (n_buf / 16) * 16 + t; i < n_buf; i += LZ_THREADS) buf[i] = src[i];
  for (int i = t; i < HASH_SIZE; i += LZ_THREADS) hash[i] = 0;
  __syncthreads();

  // Adler-32 of the segment: contiguous pieces of PER_THREAD bytes, combined in order
  {
    const int a = t * PER_THREAD, b = min(a + PER_THREAD, n_seg);
    uint32_t s1 = 1, s2 = 0;
    for (int i = a; i < b; i++) {
      s1 += buf[n_win + i];
      s2 += s1;
    }
    uint32_t ad = (s1 % ADLER_BASE) | ((s2 % ADLER_BASE) << 16);
    uint32_t len = (uint32_t)max(0, b - a);
    const int lane = t & 31;
    for (int o = 1; o < 32; o <<= 1) {   // lane l combines with lane l + o (ordered tree)
      const uint32_t ad2 = __shfl_down_sync(FULL, ad, o), len2 = __shfl_down_sync(FULL, len, o);
      if ((lane & (2 * o - 1)) == 0) {
        ad = adler_combine(ad, ad2, len2);
        len += len2;
      }
    }
    if (lane == 0) red[t >> 5] = ad, red2[t >> 5] = len;
    __syncthreads();
    if (t < 32) {
      ad = red[t], len = red2[t];
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t ad2 = __shfl_down_sync(FULL, ad, o), len2 = __shfl_down_sync(FULL, len, o);
        if ((t & (2 * o - 1)) == 0) {
          ad = adler_combine(ad, ad2, len2);
          len += len2;
        }
      }
      if (t == 0) meta.adler = ad, meta.n = (uint32_t)n_seg;
    }
  }
  // the window's 3-byte prefixes (latest position + 1 per hash)
  for (int q = t; q < n_win; q += LZ_THREADS)
    if (q + 2 < n_buf) atomicMax(hash + hash3(buf, q), (uint32_t)q + 1);
  __syncthreads();

  // matches, 1024 positions per round: the hash table holds the positions before the round, round_hash[] this
  // round's own prefixes (the nearest earlier one of the same hash, up to NEAR_SCAN positions back, is a candidate)
  const uint32_t row_dist = 3u * (uint32_t)W + 1u;
  for (int r = 0; r < PER_THREAD; r++) {
    const int p = r * LZ_THREADS + t;
    const uint32_t at = (uint32_t)(n_win + p);
    const bool hashed = p < n_seg && at + 2 < (uint32_t)n_buf;
    const uint32_t h = hashed ? hash3(buf, at) : 0u;
    round_hash[t] = hashed ? (uint16_t)h : (uint16_t)0xffff;
    __syncthreads();
    if (p < n_seg) {
      const int maxlen = min(MAX_MATCH, n_seg - p);
      int best = 0;
      uint32_t bd = 0;
      if (maxlen >= 3) {
        uint32_t near = 0;
        for (int j = t - 1; j >= max(0, t - NEAR_SCAN); j--)
          if (round_hash[j] == h) {
            near = (uint32_t)(t - j);
            break;
          }
        const uint32_t hc = hash[h];
        const uint32_t cand[5] = {1u, 3u, near, row_dist, hc ? at - (hc - 1) : 0u};
#pragma unroll
        for (int c = 0; c < 5; c++) {
          const uint32_t d = cand[c];
          if (d == 0 || d > (uint32_t)PNG_WIN || d > at || best == maxlen) continue;
          int m = match_len(buf, buf32, at, d, maxlen);
          if (m < min_match(d)) m = 0;
          if (m > best) best = m, bd = d;   // ties: the earlier candidate
        }
      }
      rec[p] = best >= 3 ? (uint32_t)best | ((bd - 1) << 9) : ((uint32_t)buf[at] << 9);
    }
    __syncthreads();
    if (hashed) atomicMax(hash + h, at + 1);
    __syncthreads();
  }

  // the greedy parse by pointer doubling: jump[p] = min(p + max(1, len), n_seg), squared 15 times; a marked position
  // marks its jump target before every squaring, so all 2^15 >= n_seg steps of the walk from 0 get marked
  for (int i = 0; i < PER_THREAD; i++) {
    const int p = i * LZ_THREADS + t;
    if (p < n_seg) {
      const int len = rec[p] & 511;
      jump[p] = (uint16_t)min(p + max(1, len), n_seg);
    }
  }
  if (t == 0) rec[0] |= MARK;
  __syncthreads();
  for (int level = 0; level < 15; level++) {
    for (int i = 0; i < PER_THREAD; i++) {
      const int p = i * LZ_THREADS + t;
      if (p < n_seg && (rec[p] & MARK)) {
        const int j = jump[p];
        if (j < n_seg) atomicOr(rec + j, MARK);
      }
    }
    __syncthreads();
    uint32_t nj[PER_THREAD / 2];
#pragma unroll
    for (int i = 0; i < PER_THREAD; i += 2) {
      uint32_t pair = 0;
#pragma unroll
      for (int h2 = 0; h2 < 2; h2++) {
        const int p = (i + h2) * LZ_THREADS + t;
        uint32_t v = (uint32_t)n_seg;
        if (p < n_seg) {
          const int j = jump[p];
          v = j < n_seg ? jump[j] : (uint32_t)n_seg;
        }
        pair |= v << (16 * h2);
      }
      nj[i / 2] = pair;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < PER_THREAD; i += 2)
#pragma unroll
      for (int h2 = 0; h2 < 2; h2++) {
        const int p = (i + h2) * LZ_THREADS + t;
        if (p < n_seg) jump[p] = (uint16_t)(nj[i / 2] >> (16 * h2));
      }
    __syncthreads();
  }

  // symbol counts of the parse
  for (int i = t; i < LIT_SYMS + DIST_SYMS + CL_SYMS; i += LZ_THREADS) (&hs.lit_freq[0])[i] = 0;
  if (t == 0) hs.extra_bits = 0;
  __syncthreads();
  {
    uint32_t extra = 0;
    for (int i = 0; i < PER_THREAD; i++) {
      const int p = t * PER_THREAD + i;
      if (p >= n_seg) break;
      const uint32_t rc = rec[p];
      if (!(rc & MARK)) continue;
      const int len = rc & 511;
      if (len == 0) {
        atomicAdd(hs.lit_freq + ((rc >> 9) & 255), 1u);
      } else {
        int sym, eb, ev;
        length_code(len, sym, eb, ev);
        atomicAdd(hs.lit_freq + sym, 1u);
        extra += eb;
        dist_code((int)((rc >> 9) & 0x7fff) + 1, sym, eb, ev);
        atomicAdd(hs.dist_freq + sym, 1u);
        extra += eb;
      }
    }
    if (extra) atomicAdd(&hs.extra_bits, extra);
  }
  if (t == 0) hs.lit_freq[256] = 1;   // end of block
  __syncthreads();

  // the dynamic codes: the tree counts (two_used may add counts that cost no data bits; lit_code / dist_code hold
  // them until the codes are made), the leaves ordered by (count, symbol) in parallel, one thread per tree
  if (t == 0 || t == 32) {
    const bool lit = t == 0;
    uint32_t* counts = lit ? hs.lit_code : hs.dist_code;
    const uint32_t* f0 = lit ? hs.lit_freq : hs.dist_freq;
    const int n = lit ? LIT_SYMS : DIST_SYMS;
    for (int i = 0; i < n; i++) counts[i] = f0[i];
    two_used(counts, n);
  }
  __syncthreads();
  if (t < LIT_SYMS || (t >= 512 && t < 512 + DIST_SYMS)) {
    const bool lit = t < LIT_SYMS;
    const uint32_t* counts = lit ? hs.lit_code : hs.dist_code;
    const int n = lit ? LIT_SYMS : DIST_SYMS, sym = lit ? t : t - 512;
    const uint32_t c = counts[sym];
    if (c) {
      int rank = 0;
      for (int u = 0; u < n; u++) rank += counts[u] != 0 && (counts[u] < c || (counts[u] == c && u < sym));
      (lit ? hs.order_a : hs.order_b)[rank] = (uint16_t)sym;
    }
  }
  __syncthreads();
  if (t == 0 || t == 32) {
    const bool lit = t == 0;
    const uint32_t* counts = lit ? hs.lit_code : hs.dist_code;
    const int n = lit ? LIT_SYMS : DIST_SYMS;
    int m = 0;
    for (int i = 0; i < n; i++) m += counts[i] != 0;
    huffman_lengths(counts, n, m, 15, lit ? hs.order_a : hs.order_b, lit ? hs.work_a : hs.work_b,
                    lit ? hs.lit_len : hs.dist_len);
  }
  __syncthreads();
  if (t == 0) {
    int hlit = LIT_SYMS, hdist = DIST_SYMS;
    while (hlit > 257 && hs.lit_len[hlit - 1] == 0) hlit--;
    while (hdist > 1 && hs.dist_len[hdist - 1] == 0) hdist--;
    // run-length code of the hlit + hdist lengths as one sequence
    auto L = [&](int i) -> int { return i < hlit ? hs.lit_len[i] : hs.dist_len[i - hlit]; };
    const int total = hlit + hdist;
    int nr = 0;
    for (int i = 0; i < CL_SYMS; i++) hs.cl_freq[i] = 0;
    int i = 0;
    while (i < total) {
      const int v = L(i);
      int run = 1;
      while (i + run < total && L(i + run) == v) run++;
      i += run;
      if (v == 0) {
        while (run >= 11) {
          const int r = min(run, 138);
          hs.rle[nr++] = (uint16_t)(18 | ((r - 11) << 5));
          hs.cl_freq[18]++;
          run -= r;
        }
        if (run >= 3) {
          hs.rle[nr++] = (uint16_t)(17 | ((run - 3) << 5));
          hs.cl_freq[17]++;
          run = 0;
        }
        for (; run > 0; run--) {
          hs.rle[nr++] = 0;
          hs.cl_freq[0]++;
        }
      } else {
        hs.rle[nr++] = (uint16_t)v;
        hs.cl_freq[v]++;
        run--;
        while (run >= 3) {
          const int r = min(run, 6);
          hs.rle[nr++] = (uint16_t)(16 | ((r - 3) << 5));
          hs.cl_freq[16]++;
          run -= r;
        }
        for (; run > 0; run--) {
          hs.rle[nr++] = (uint16_t)v;
          hs.cl_freq[v]++;
        }
      }
    }
    uint32_t* clf = hs.cl_code;   // the counts, until the codes are made
    for (int c = 0; c < CL_SYMS; c++) clf[c] = hs.cl_freq[c];
    two_used(clf, CL_SYMS);
    int m = 0;
    for (int s2 = 0; s2 < CL_SYMS; s2++) {   // insertion by (count, symbol)
      if (clf[s2] == 0) continue;
      int j = m++;
      while (j > 0 && clf[hs.order_b[j - 1]] > clf[s2]) {
        hs.order_b[j] = hs.order_b[j - 1];
        j--;
      }
      hs.order_b[j] = (uint16_t)s2;
    }
    huffman_lengths(clf, CL_SYMS, m, 7, hs.order_b, hs.work_b, hs.cl_len);
    int hclen = CL_SYMS;
    while (hclen > 4 && hs.cl_len[CL_ORDER[hclen - 1]] == 0) hclen--;
    hs.n_rle = nr, hs.hlit = hlit, hs.hdist = hdist, hs.hclen = hclen;
    // exact costs
    uint64_t header = 3 + 5 + 5 + 4 + 3 * hclen;
    for (int r = 0; r < nr; r++) {
      const int sym = hs.rle[r] & 31;
      header += hs.cl_len[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
    }
    uint64_t dyn = header + hs.extra_bits, fix = 3 + hs.extra_bits;
    for (int c = 0; c < LIT_SYMS; c++) {
      dyn += (uint64_t)hs.lit_freq[c] * hs.lit_len[c];
      fix += (uint64_t)hs.lit_freq[c] * fixed_lit_len(c);
    }
    for (int c = 0; c < DIST_SYMS; c++) {
      dyn += (uint64_t)hs.dist_freq[c] * hs.dist_len[c];
      fix += (uint64_t)hs.dist_freq[c] * 5;
    }
    hs.header_bits = (uint32_t)header;
    hs.use_fixed = fix <= dyn;   // ties: the fixed block
    const uint64_t huff = hs.use_fixed ? fix : dyn;
    const uint64_t stored_max = 42 + 8 * (uint64_t)n_seg;
    hs.huff_bits = huff <= stored_max ? (uint32_t)huff : NO_HUFF;
    meta.huff_bits = hs.huff_bits;
    // the codes of the block to render
    if (hs.use_fixed) {
      for (int c = 0; c < LIT_SYMS; c++) {
        const int len = fixed_lit_len(c);
        const uint32_t code = c < 144 ? 0x30 + c : c < 256 ? 0x190 + (c - 144) : c < 280 ? c - 256 : 0xc0 + (c - 280);
        hs.lit_code[c] = bit_reverse(code, len) | ((uint32_t)len << 16);
      }
      for (int c = 0; c < DIST_SYMS; c++) hs.dist_code[c] = bit_reverse((uint32_t)c, 5) | (5u << 16);
    } else {
      canonical_codes(hs.lit_len, LIT_SYMS, hs.lit_code);
      canonical_codes(hs.dist_len, DIST_SYMS, hs.dist_code);
      canonical_codes(hs.cl_len, CL_SYMS, hs.cl_code);
    }
  }
  __syncthreads();
  if (hs.huff_bits == NO_HUFF) return;   // a stored block in any case: png_pack_kernel copies the bytes

  // render: each thread's PER_THREAD positions are contiguous, so one scan of per-thread bit counts places them
  uint32_t* stage = l.stage + ((int64_t)k * l.S + s) * STAGE_WORDS;
  const uint32_t words = (hs.huff_bits + 31) / 32;
  for (uint32_t i = t; i < words + 2; i += LZ_THREADS) bits[i] = 0;
  auto sym_bits = [&](uint32_t rc, uint64_t& v, int& nb) {
    const int len = rc & 511;
    if (len == 0) {
      const uint32_t c = hs.lit_code[(rc >> 9) & 255];
      v = c & 0xffff, nb = (int)(c >> 16);
      return;
    }
    int sym, eb, ev;
    length_code(len, sym, eb, ev);
    uint32_t c = hs.lit_code[sym];
    v = c & 0xffff, nb = (int)(c >> 16);
    v |= (uint64_t)ev << nb, nb += eb;
    dist_code((int)((rc >> 9) & 0x7fff) + 1, sym, eb, ev);
    c = hs.dist_code[sym];
    v |= (uint64_t)(c & 0xffff) << nb, nb += (int)(c >> 16);
    v |= (uint64_t)ev << nb, nb += eb;
  };
  uint32_t mine = 0;
  for (int i = 0; i < PER_THREAD; i++) {
    const int p = t * PER_THREAD + i;
    if (p >= n_seg) break;
    if (rec[p] & MARK) {
      uint64_t v;
      int nb;
      sym_bits(rec[p], v, nb);
      mine += nb;
    }
  }
  uint32_t body = 0;
  const uint32_t head = hs.use_fixed ? 3u : hs.header_bits;
  uint32_t at = head + block_exclusive_scan(mine, red, &body);   // (the scan's barriers order the zeroing too)
  for (int i = 0; i < PER_THREAD; i++) {
    const int p = t * PER_THREAD + i;
    if (p >= n_seg) break;
    if (rec[p] & MARK) {
      uint64_t v;
      int nb;
      sym_bits(rec[p], v, nb);
      put_bits(bits, at, v, nb);
      at += nb;
    }
  }
  if (t == 0) {
    put_bits(bits, head + body, hs.lit_code[256] & 0xffff, (int)(hs.lit_code[256] >> 16));   // end of block
    if (hs.use_fixed) {
      put_bits(bits, 0, 1u << 1, 3);   // BFINAL 0 (png_pack_kernel sets it on the last block), BTYPE 01
    } else {
      uint32_t o = 0;
      put_bits(bits, o, 2u << 1, 3), o += 3;   // BTYPE 10
      put_bits(bits, o, hs.hlit - 257, 5), o += 5;
      put_bits(bits, o, hs.hdist - 1, 5), o += 5;
      put_bits(bits, o, hs.hclen - 4, 4), o += 4;
      for (uint32_t i = 0; i < hs.hclen; i++) put_bits(bits, o, hs.cl_len[CL_ORDER[i]], 3), o += 3;
      for (uint32_t r = 0; r < hs.n_rle; r++) {
        const int sym = hs.rle[r] & 31, ev = hs.rle[r] >> 5;
        const uint32_t c = hs.cl_code[sym];
        put_bits(bits, o, c & 0xffff, (int)(c >> 16)), o += c >> 16;
        const int eb = sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0;
        put_bits(bits, o, (uint32_t)ev, eb), o += eb;
      }
    }
  }
  __syncthreads();
  for (uint32_t i = t; i < words; i += LZ_THREADS) stage[i] = bits[i];
}

__global__ void __launch_bounds__(32) png_offsets_kernel(int64_t* __restrict__ out_len, Layout l) {
  const int k = blockIdx.x;
  if (threadIdx.x != 0) return;
  SegMeta* seg = l.seg + (int64_t)k * l.S;
  int64_t off = 0;
  uint32_t adler = 1;
  for (int64_t s = 0; s < l.S; s++) {
    SegMeta& m = seg[s];
    const int64_t pad = (8 - ((off + 3) & 7)) & 7;
    const int64_t stored = 3 + pad + 32 + 8 * (int64_t)m.n;
    const bool st = m.huff_bits == NO_HUFF || stored <= (int64_t)m.huff_bits;   // ties: the stored block
    m.stored = st;
    m.off = off;
    off += st ? stored : (int64_t)m.huff_bits;
    adler = adler_combine(adler, m.adler, m.n);
  }
  const int64_t idat = 2 + (off + 7) / 8 + 4;
  l.view[k].total_bits = off;
  l.view[k].adler = adler;
  l.view[k].idat_len = (uint32_t)idat;
  out_len[k] = 8 + 25 + 12 + idat + 12;
}

// bits [32 w, 32 w + 32) of the deflate stream that segment `m` contributes
__device__ __forceinline__ uint32_t segment_word(const SegMeta& m, bool last, int64_t w, const uint32_t* stage,
                                                 const uint8_t* bytes) {
  const int64_t lo = 32 * w;
  if (!m.stored) {
    const int64_t bits = m.huff_bits;
    uint32_t v = 0;
    const int64_t rel = lo - m.off;   // bit rel of the block lands on bit 0 of the word
    if (rel >= 0) {
      const int64_t i = rel >> 5;
      const int sh = (int)(rel & 31);
      const uint32_t a = i * 32 < bits ? stage[i] : 0u, b = (i + 1) * 32 < bits ? stage[i + 1] : 0u;
      v = sh ? __funnelshift_r(a, b, sh) : a;
    } else {
      v = stage[0] << (-rel);   // -rel < 32: this word holds the block's first bit
    }
    // the block's bits beyond its length are zero in the staging area; bits before it are shifted out
    if (last && m.off >= lo && m.off < lo + 32) v |= 1u << (m.off - lo);
    return v;
  }
  // a stored block: header bits (BFINAL, BTYPE 00), padding to a byte, LEN, NLEN, the bytes
  const int64_t data_bit = ((m.off + 3 + 7) / 8) * 8;   // LEN's first bit
  uint32_t v = 0;
#pragma unroll
  for (int b = 0; b < 4; b++) {
    const int64_t g = lo + 8 * b;   // this byte's first bit
    uint32_t byte = 0;
    if (g >= data_bit) {
      const int64_t i = (g - data_bit) / 8;
      if (i < 4) {
        const uint32_t len = m.n, nlen = ~m.n & 0xffff;
        byte = i == 0 ? len & 255 : i == 1 ? (len >> 8) & 255 : i == 2 ? nlen & 255 : (nlen >> 8) & 255;
      } else if (i - 4 < (int64_t)m.n) {
        byte = bytes[i - 4];
      }
    } else if (last && m.off >= g && m.off < g + 8) {
      byte = 1u << (m.off - g);   // BFINAL; BTYPE 00 and the padding are zero
    }
    v |= byte << (8 * b);
  }
  return v;
}

__global__ void __launch_bounds__(256) png_pack_kernel(Layout l) {
  const int s = blockIdx.x, k = blockIdx.y;
  const SegMeta m = l.seg[(int64_t)k * l.S + s];
  const bool last = s == l.S - 1;
  const int64_t nbits = m.stored ? ((m.off + 3 + 7) / 8) * 8 + 32 + 8 * (int64_t)m.n - m.off : (int64_t)m.huff_bits;
  const int64_t w0 = m.off >> 5, w1 = (m.off + nbits - 1) >> 5;
  uint32_t* defl = l.defl + k * l.defl_words;
  const uint32_t* stage = l.stage + ((int64_t)k * l.S + s) * STAGE_WORDS;
  const uint8_t* bytes = l.filt + k * l.filt_stride + (int64_t)s * PNG_SEG;
  for (int64_t w = w0 + threadIdx.x; w <= w1; w += blockDim.x) {
    const uint32_t v = segment_word(m, last, w, stage, bytes);
    if (w == w0 || w == w1) atomicOr(defl + w, v);   // shared with the neighbouring blocks
    else defl[w] = v;
  }
}

__device__ void crc_tables(uint32_t* table, uint32_t* x2n) {
  for (int t = threadIdx.x; t < 256; t += blockDim.x) {
    uint32_t c = t;
    for (int j = 0; j < 8; j++) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
    table[t] = c;
  }
  if (threadIdx.x == 0) {
    uint32_t p = 1u << 30;   // x^1
    x2n[0] = p;
    for (int i = 1; i < 32; i++) x2n[i] = p = crc_multmodp(p, p);
  }
  __syncthreads();
}

// in-order tree combine of n (crc, len) pairs in shared memory (n a power of two <= blockDim.x); the result in [0]
__device__ void crc_tree(uint32_t* crc, uint64_t* len, int n, const uint32_t* x2n) {
  const int t = threadIdx.x;
  for (int o = 1; o < n; o <<= 1) {
    if (t < n && (t & (2 * o - 1)) == 0) {
      crc[t] = crc_combine(crc[t], crc[t + o], len[t + o], x2n);
      len[t] += len[t + o];
    }
    __syncthreads();
  }
}

// One CTA per ASM_CHUNK bytes of the IDAT chunk's type and data ("IDAT" || 78 01 || deflate bytes || Adler-32): the
// bytes into the file, and the piece's CRC-32 into the scratch.
__global__ void __launch_bounds__(256) png_assemble_kernel(uint8_t* __restrict__ out, int64_t out_stride, Layout l) {
  __shared__ uint32_t table[256], x2n[32], crc_part[256];
  __shared__ uint64_t len_part[256];
  const int c = blockIdx.x, k = blockIdx.y, t = threadIdx.x;
  const ViewMeta vm = l.view[k];
  const int64_t deflate_bytes = (vm.total_bits + 7) / 8, total = 4 + (int64_t)vm.idat_len;
  const int64_t c0 = (int64_t)c * ASM_CHUNK;
  if (c0 >= total) return;
  crc_tables(table, x2n);
  const uint8_t* defl = reinterpret_cast<const uint8_t*>(l.defl + k * l.defl_words);
  uint8_t* idat = out + k * out_stride + 8 + 25 + 4;   // the chunk's type
  const int64_t per = ASM_CHUNK / 256;
  const int64_t a = min(c0 + t * per, total), b = min(a + per, total);
  uint32_t crc = 0xffffffffu;
  for (int64_t i = a; i < b; i++) {
    uint32_t v;
    if (i >= 6 && i < 6 + deflate_bytes) v = defl[i - 6];
    else if (i < 4) v = (0x49444154u >> (8 * (3 - i))) & 255;   // "IDAT"
    else if (i == 4) v = 0x78;                                 // CMF: deflate, 32 KiB window
    else if (i == 5) v = 0x01;                                 // FLG: check bits, no dictionary
    else v = (vm.adler >> (8 * (3 - (i - 6 - deflate_bytes)))) & 255;
    idat[i] = (uint8_t)v;
    crc = table[(crc ^ v) & 255] ^ (crc >> 8);
  }
  crc_part[t] = crc ^ 0xffffffffu;
  len_part[t] = (uint64_t)(b - a);
  __syncthreads();
  crc_tree(crc_part, len_part, 256, x2n);
  if (t == 0) l.crc[(int64_t)k * l.chunks + c] = make_uint2(crc_part[0], (uint32_t)len_part[0]);
}

// One CTA per view: the signature, IHDR, the IDAT's length and CRC-32 (its pieces' CRCs combined in order), IEND.
__global__ void __launch_bounds__(1024) png_finish_kernel(int H, int W, uint8_t* __restrict__ out, int64_t out_stride,
                                                          Layout l) {
  __shared__ uint32_t table[256], x2n[32], crc_part[1024];
  __shared__ uint64_t len_part[1024];
  const int k = blockIdx.x, t = threadIdx.x;
  const ViewMeta vm = l.view[k];
  const int64_t D = vm.idat_len, pieces = (4 + D + ASM_CHUNK - 1) / ASM_CHUNK;
  crc_tables(table, x2n);
  // each thread combines a run of consecutive pieces, then the runs combine in a tree
  const int64_t per = (pieces + 1023) / 1024, a = min((int64_t)t * per, pieces), b = min(a + per, pieces);
  uint32_t crc = 0;
  uint64_t len = 0;
  for (int64_t i = a; i < b; i++) {
    const uint2 e = l.crc[(int64_t)k * l.chunks + i];
    crc = len ? crc_combine(crc, e.x, e.y, x2n) : e.x;
    len += e.y;
  }
  crc_part[t] = crc;
  len_part[t] = len;
  __syncthreads();
  crc_tree(crc_part, len_part, 1024, x2n);
  if (t == 0) {
    uint8_t* f = out + k * out_stride;
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    for (int i = 0; i < 8; i++) f[i] = sig[i];
    uint8_t* ih = f + 8;
    put_be32(ih, 13);
    const uint8_t type[4] = {'I', 'H', 'D', 'R'};
    for (int i = 0; i < 4; i++) ih[4 + i] = type[i];
    put_be32(ih + 8, (uint32_t)W);
    put_be32(ih + 12, (uint32_t)H);
    ih[16] = 8, ih[17] = 2, ih[18] = 0, ih[19] = 0, ih[20] = 0;   // 8 bits, RGB, deflate, adaptive filters, no interlace
    uint32_t hc = 0xffffffffu;
    for (int i = 4; i < 21; i++) hc = table[(hc ^ ih[i]) & 255] ^ (hc >> 8);
    put_be32(ih + 21, hc ^ 0xffffffffu);
    uint8_t* idat = f + 8 + 25;
    put_be32(idat, (uint32_t)D);
    put_be32(idat + 8 + D, crc_part[0]);
    uint8_t* end = idat + 12 + D;
    put_be32(end, 0);
    const uint8_t iend[4] = {'I', 'E', 'N', 'D'};
    for (int i = 0; i < 4; i++) end[4 + i] = iend[i];
    put_be32(end + 8, 0xae426082u);
  }
}

__global__ void __launch_bounds__(256) png_copy_kernel(const uint8_t* __restrict__ src, int64_t src_stride,
                                                       const int64_t* __restrict__ src_len,
                                                       const int32_t* __restrict__ flag, uint8_t* dst,
                                                       int64_t dst_stride, int64_t* dst_len) {
  const int k = blockIdx.y;
  const bool over = flag != nullptr && *flag != 0;
  const int64_t n = over ? -1 : src_len[k];
  if (blockIdx.x == 0 && threadIdx.x == 0) dst_len[k] = n;
  if (n <= 0) return;
  const uint4* s = reinterpret_cast<const uint4*>(src + k * src_stride);
  uint4* d = reinterpret_cast<uint4*>(dst + k * dst_stride);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n + 15) / 16; i += (int64_t)gridDim.x * blockDim.x)
    d[i] = s[i];
}

}  // namespace

int64_t png_bound(int H, int W) {
  if (H <= 0 || W <= 0 || W > (INT32_MAX - 1) / 3) return -1;
  const int64_t row = 3 * (int64_t)W + 1;
  if ((int64_t)H > ((int64_t)INT32_MAX - 1024) / row) return -1;
  const int64_t n = filtered_bytes(H, W), bound = 63 + n + 6 * segments_of(n);
  return bound - 45 - 12 <= (int64_t)INT32_MAX ? bound : -1;   // the IDAT length is a 31-bit field
}

size_t png_scratch_bytes(int64_t views, int H, int W) {
  if (views <= 0 || views > 65535 || png_bound(H, W) < 0) return 0;
  return carve(nullptr, views, H, W).bytes;
}

void launch_png_encode(int views, int H, int W, const uint8_t* rgb, void* scratch, uint8_t* out, int64_t out_stride,
                       int64_t* out_len, cudaStream_t stream) {
  cudaFuncSetAttribute(png_lz_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LZ_SMEM);
  const Layout l = carve(scratch, views, H, W);
  const int64_t n = filtered_bytes(H, W);
  png_filter_kernel<<<dim3((unsigned)H, (unsigned)views), 256, 0, stream>>>(H, W, rgb, l);
  count_launch();
  png_lz_kernel<<<dim3((unsigned)l.S, (unsigned)views), LZ_THREADS, LZ_SMEM, stream>>>(W, n, l);
  count_launch();
  png_offsets_kernel<<<(unsigned)views, 32, 0, stream>>>(out_len, l);
  count_launch();
  png_pack_kernel<<<dim3((unsigned)l.S, (unsigned)views), 256, 0, stream>>>(l);
  count_launch();
  png_assemble_kernel<<<dim3((unsigned)l.chunks, (unsigned)views), 256, 0, stream>>>(out, out_stride, l);
  count_launch();
  png_finish_kernel<<<(unsigned)views, 1024, 0, stream>>>(H, W, out, out_stride, l);
  count_launch();
}

void launch_png_copy(int views, const uint8_t* src, int64_t src_stride, const int64_t* src_len, const int32_t* flag,
                     uint8_t* dst, int64_t dst_stride, int64_t* dst_len, cudaStream_t stream) {
  const int64_t words = (src_stride + 15) / 16;
  const unsigned blocks = (unsigned)max((int64_t)1, min((int64_t)64, (words + 255) / 256));
  png_copy_kernel<<<dim3(blocks, (unsigned)views), 256, 0, stream>>>(src, src_stride, src_len, flag, dst, dst_stride,
                                                                     dst_len);
  count_launch();
}

}  // namespace gab
