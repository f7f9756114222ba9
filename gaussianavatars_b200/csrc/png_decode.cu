// png_decode.cu -- PNG files read on the device (gab200_png_decode_scratch_bytes / gab200_png_decode): the IDAT data
// of F files of one size, 8-bit RGB or RGBA, not interlaced, inflated and unfiltered into (F, H, W, 3 or 4) bytes.
//
// Two kernels, each named for a trace, one warp per file and PNG_DEC_WARPS files per CTA:
//   png_inflate_kernel   the file's zlib stream, RFC 1950/1951 with zlib's validity rules (inflate.c, inftrees.c;
//                        oracle/inflate.py restates them), into the file's scratch: the filtered stream, H rows of
//                        1 + W c bytes, which is also the 32 KiB window.  Every lane runs the same serial decode on
//                        the same 64-bit bit buffer, so the control flow stays uniform; lane 0 writes literals, the
//                        whole warp writes each match (out[p + i] = out[p - d + i mod d], right for every overlap) and
//                        each stored block.  Each dynamic block's tables are built by the warp in its shared memory:
//                        a primary table indexed by the next 9 (literal/length) or 6 (distance) bits, and sub-tables
//                        for longer codes sized as zlib's inflate_table sizes them (so within zlib's ENOUGH_LENS 852
//                        and ENOUGH_DISTS 592 entries); each entry decodes itself by canonical-code arithmetic, so
//                        the lanes fill the table in parallel.  The fixed tables are built once per CTA.  Then the
//                        Adler-32 of the stream: per-lane sums over 32 slices, combined with adler_combine.
//   png_unfilter_kernel  the five row filters undone as a wavefront: lane i takes row r + i one pixel behind lane
//                        i - 1, so the up and up-left pixels arrive by __shfl_up_sync from lane i - 1's last two steps
//                        and 32 rows advance together.  Lane 31 writes its raw row back into the scratch in place,
//                        where lane 0 of the next 32 rows reads it as its row above.  Writes RGBA (alpha 255 for an
//                        RGB file) or RGB.
//
// Safety: the bytes come from files.  Every read of the stream is bounded by the file's length (bytes past it read
// as zero, and a decode that consumes one of them ends TRUNCATED); every write lies in the file's own scratch slot
// (a literal or match is refused before it would pass H (1 + W c) bytes) or its own output image; every distance is
// checked against the bytes already written; HLIT, HDIST and every repeat are checked before they index the length
// array.  A file's status is the first error in stream order (include/gab200_rasterizer.h, gab200_png_status).
#include "common.cuh"
#include "deflate.cuh"
#include "kernels.cuh"

namespace gab {

namespace {

constexpr int PNG_DEC_WARPS = 4;
constexpr unsigned FULL = 0xffffffffu;
constexpr int LIT_ROOT = 9, DIST_ROOT = 6, CL_ROOT = 7;
constexpr int LIT_ENOUGH = 852, DIST_ENOUGH = 592, CL_ENOUGH = 1 << CL_ROOT;   // zlib's inftrees.h bounds

// a table entry: value (symbol or sub-table offset) in bits 0..15, bit count in 16..23, kind in 24..31
constexpr uint32_t K_SYM = 0, K_LINK = 1, K_BAD = 2;
__device__ __forceinline__ uint32_t entry(uint32_t kind, uint32_t bits, uint32_t val) {
  return (kind << 24) | (bits << 16) | val;
}

// RFC 1951 3.2.5: base and extra bits of length codes 257..285 and distance codes 0..29
__constant__ uint16_t LEN_BASE[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t LEN_EXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t DIST_BASE[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,    65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t DIST_EXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

// canonical-code bookkeeping of one table build
struct TabWork {
  int32_t cnt[16], first[16], offs[16], run[16];
  uint16_t sorted[288];   // symbols ordered by (length, symbol)
};

struct WarpSmem {
  uint32_t lit[LIT_ENOUGH];
  uint32_t dist[DIST_ENOUGH];
  uint32_t cl[CL_ENOUGH];
  TabWork w;
  uint8_t lens[320];      // the code lengths of a block: HLIT + HDIST <= 316
};

struct CtaSmem {
  uint32_t fixed_lit[1 << LIT_ROOT];
  uint32_t fixed_dist[1 << DIST_ROOT];
  WarpSmem warp[PNG_DEC_WARPS];
};

__device__ __forceinline__ uint32_t rev(uint32_t v, int bits) { return __brev(v) >> (32 - bits); }

// The symbol of canonical code `code` of `len` bits, or -1 (len <= 15)
__device__ __forceinline__ int canonical(const TabWork& w, uint32_t code, int len) {
  const uint32_t i = code - (uint32_t)w.first[len];
  return i < (uint32_t)w.cnt[len] ? w.sorted[w.offs[len] + i] : -1;
}

// Builds the decode table of the n code lengths lens[0 .. n) with a primary table of 2^root entries (root >= 5) and
// sub-tables after it, in at most `cap` entries.  False for an over-subscribed code and for an incomplete one, except
// (allow_incomplete) an empty code or a single code of length 1, whose unused codes decode as K_BAD of 1 bit.
// Called by a whole warp; lens is in shared memory.
__device__ bool build_table(const uint8_t* lens, int n, int root, uint32_t* table, int cap, bool allow_incomplete,
                            TabWork& w, int lane) {
  if (lane < 16) w.cnt[lane] = 0, w.run[lane] = 0;
  __syncwarp();
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + lane;
    const int len = s < n ? lens[s] : 0;
    const unsigned m = __match_any_sync(FULL, len);
    if (len && lane == __ffs(m) - 1) w.cnt[len] += __popc(m);
  }
  __syncwarp();
  int left = 1, code = 0, off = 0, maxl = 0;
  for (int len = 1; len <= 15; len++) {
    const int c = w.cnt[len];
    left = 2 * left - c;
    if (left < 0) break;
    if (lane == len) w.first[len] = code, w.offs[len] = off;
    code = (code + c) << 1;
    off += c;
    if (c) maxl = len;
  }
  if (left < 0) return false;                                     // over-subscribed
  if (left > 0 && !(allow_incomplete && maxl <= 1)) return false;  // incomplete
  __syncwarp();
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + lane;
    const int len = s < n ? lens[s] : 0;
    const unsigned m = __match_any_sync(FULL, len);
    const int base = len ? w.run[len] : 0;
    if (len) w.sorted[w.offs[len] + base + __popc(m & ((1u << lane) - 1))] = (uint16_t)s;
    __syncwarp();
    if (len && lane == __ffs(m) - 1) w.run[len] += __popc(m);
    __syncwarp();
  }
  // primary entries, and the sub-table each prefix of longer codes links to
  const int size = 1 << root;
  int next = size;
  for (int e0 = 0; e0 < size; e0 += 32) {
    const uint32_t v = rev(e0 + lane, root);   // the next root bits as a code, first bit most significant
    uint32_t ent = entry(K_BAD, 1, 0);
    int sub = 0;
    bool found = false;
    for (int len = 1; len <= min(maxl, root) && !found; len++) {
      const int s = canonical(w, v >> (root - len), len);
      if (s >= 0) ent = entry(K_SYM, len, s), found = true;
    }
    if (!found && maxl > root) {
      // the sub-table spans the longest code under this prefix (zlib's sizing for a complete code)
      for (int len = maxl; len > root && !sub; len--) {
        const uint32_t lo = v << (len - root), hi = lo + (1u << (len - root));
        const uint32_t f = w.first[len], fe = f + w.cnt[len];
        if (w.cnt[len] && lo < fe && f < hi) sub = len - root;
      }
    }
    const int sz = sub ? 1 << sub : 0;
    int incl = sz;
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(FULL, incl, o);
      if (lane >= o) incl += t;
    }
    if (sub) ent = entry(K_LINK, sub, min(next + incl - sz, 0xffff));
    next += __shfl_sync(FULL, incl, 31);
    table[e0 + lane] = ent;
  }
  if (next > cap) return false;   // cannot happen for a complete code (zlib's ENOUGH bounds); never written past cap
  __syncwarp();
  for (int e0 = 0; e0 < size; e0 += 32) {
    const uint32_t mine = table[e0 + lane];
    unsigned links = __ballot_sync(FULL, (mine >> 24) == K_LINK);
    while (links) {
      const int j = __ffs(links) - 1;
      links &= links - 1;
      const uint32_t le = __shfl_sync(FULL, mine, j);
      const uint32_t v = rev(e0 + j, root);
      const int sub = (le >> 16) & 255, at = le & 0xffff;
      for (int k = lane; k < (1 << sub); k += 32) {
        const uint32_t full = (v << sub) | rev(k, sub);
        uint32_t ent = entry(K_BAD, sub, 0);
        for (int len = root + 1; len <= root + sub; len++) {
          const int s = canonical(w, full >> (root + sub - len), len);
          if (s >= 0) {
            ent = entry(K_SYM, len - root, s);
            break;
          }
        }
        table[at + k] = ent;
      }
    }
  }
  __syncwarp();
  return true;
}

// The entry the low bits of buf select, and its bit count
__device__ __forceinline__ uint32_t lookup(const uint32_t* t, int root, uint64_t buf, int& used) {
  uint32_t e = t[buf & ((1u << root) - 1)];
  if ((e >> 24) == K_LINK) {
    const int sub = (e >> 16) & 255;
    e = t[(e & 0xffff) + ((uint32_t)(buf >> root) & ((1u << sub) - 1))];
    used = root + ((e >> 16) & 255);
    return e;
  }
  used = (e >> 16) & 255;
  return e;
}

// LSB-first bit reader over one file's stream; bytes past its end read as zero
struct Bits {
  const uint8_t* p;
  int64_t len;    // bytes of the stream
  int64_t next;   // next byte to load
  uint64_t buf;
  int cnt;        // bits in buf
  __device__ __forceinline__ void refill() {   // to at least 32 bits
    if (cnt < 32) {
      uint32_t w = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) w |= (next + k < len ? (uint32_t)p[next + k] : 0u) << (8 * k);
      buf |= (uint64_t)w << cnt;
      cnt += 32;
      next += 4;
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)buf & ((1u << n) - 1); }
  __device__ __forceinline__ void drop(int n) { buf >>= n, cnt -= n; }
  __device__ __forceinline__ int64_t pos() const { return next * 8 - cnt; }   // bits consumed
  __device__ __forceinline__ bool over() const { return pos() > len * 8; }
};

__device__ __forceinline__ void fixed_lengths(uint8_t* lens, int lane) {
  for (int s = lane; s < 288; s += 32) lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
  __syncwarp();
}

// Reads a dynamic block's header and builds its tables; GAB200_PNG_OK or the first error
__device__ int dynamic_header(Bits& in, WarpSmem& ws, int lane) {
  in.refill();
  const int hlit = in.peek(5) + 257, hdist = ((in.buf >> 5) & 31) + 1, hclen = ((in.buf >> 10) & 15) + 4;
  in.drop(14);
  if (in.over()) return GAB200_PNG_TRUNCATED;
  if (hlit > 286 || hdist > 30) return GAB200_PNG_CODE_LENGTHS;
  if (lane < 19) ws.lens[lane] = 0;
  __syncwarp();
  for (int i = 0; i < hclen; i++) {
    in.refill();
    if (lane == 0) ws.lens[CL_ORDER[i]] = in.peek(3);
    in.drop(3);
  }
  if (in.over()) return GAB200_PNG_TRUNCATED;
  __syncwarp();
  if (!build_table(ws.lens, 19, CL_ROOT, ws.cl, CL_ENOUGH, false, ws.w, lane)) return GAB200_PNG_CODE_LENGTHS;
  const int total = hlit + hdist;
  int i = 0, prev = 0;
  while (i < total) {
    in.refill();
    int used;
    const int sym = lookup(ws.cl, CL_ROOT, in.buf, used) & 0xffff;   // complete, at most 7 bits: always a symbol
    in.drop(used);
    if (in.over()) return GAB200_PNG_TRUNCATED;
    if (sym < 16) {
      if (lane == 0) ws.lens[i] = sym;
      prev = sym;
      i++;
      continue;
    }
    int rep, val;
    if (sym == 16) {
      rep = 3 + in.peek(2), val = prev;
      in.drop(2);
    } else if (sym == 17) {
      rep = 3 + in.peek(3), val = 0;
      in.drop(3);
    } else {
      rep = 11 + in.peek(7), val = 0;
      in.drop(7);
    }
    if (in.over()) return GAB200_PNG_TRUNCATED;
    if (sym == 16 && i == 0) return GAB200_PNG_CODE_LENGTHS;
    if (i + rep > total) return GAB200_PNG_CODE_LENGTHS;
    for (int k = lane; k < rep; k += 32) ws.lens[i + k] = val;
    i += rep;
    prev = val;
  }
  __syncwarp();
  if (ws.lens[256] == 0) return GAB200_PNG_CODE_LENGTHS;
  if (!build_table(ws.lens, hlit, LIT_ROOT, ws.lit, LIT_ENOUGH, true, ws.w, lane)) return GAB200_PNG_CODE_LENGTHS;
  if (!build_table(ws.lens + hlit, hdist, DIST_ROOT, ws.dist, DIST_ENOUGH, true, ws.w, lane))
    return GAB200_PNG_CODE_LENGTHS;
  return GAB200_PNG_OK;
}

// The Adler-32 of p[0 .. n) (p 16-byte aligned): each lane sums one 16-byte aligned slice, in order-combined sums
__device__ uint32_t warp_adler(const uint8_t* p, int64_t n, int lane) {
  const int64_t chunk = ((n + 31) / 32 + 15) & ~int64_t(15);
  const int64_t b = min(n, lane * chunk), e = min(n, b + chunk);
  uint32_t s1 = 1, s2 = 0;
  for (int64_t i = b; i < e;) {
    const int64_t stop = min(e, i + 5536);   // 16-byte steps within zlib's NMAX = 5552 before the sums are reduced
    for (; i + 16 <= stop; i += 16) {
      const uint4 v = *reinterpret_cast<const uint4*>(p + i);
      const uint32_t words[4] = {v.x, v.y, v.z, v.w};
      const uint32_t weights[4] = {0x0D0E0F10u, 0x090A0B0Cu, 0x05060708u, 0x01020304u};
      uint32_t sum = 0, wsum = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) sum = __dp4a(words[k], 0x01010101u, sum), wsum = __dp4a(words[k], weights[k], wsum);
      s2 += 16 * s1 + wsum;
      s1 += sum;
    }
    for (; i < stop; i++) s1 += p[i], s2 += s1;
    s1 %= ADLER_BASE;
    s2 %= ADLER_BASE;
  }
  const uint32_t mine = (s2 << 16) | s1, mlen = (uint32_t)(e - b);
  uint32_t a = 1;
  for (int j = 0; j < 32; j++) a = adler_combine(a, __shfl_sync(FULL, mine, j), __shfl_sync(FULL, mlen, j));
  return a;
}

// Inflates one file's stream into dst (n bytes expected); GAB200_PNG_OK or the first error
__device__ int inflate_file(Bits& in, uint8_t* dst, int64_t n, const CtaSmem& sm, WarpSmem& ws, int lane) {
  in.refill();
  const uint32_t cmf = in.peek(8), flg = (in.buf >> 8) & 255;
  in.drop(16);
  if (in.over()) return GAB200_PNG_TRUNCATED;
  if ((cmf * 256 + flg) % 31 != 0 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 32)) return GAB200_PNG_ZLIB_HEADER;
  int64_t out = 0;
  bool last = false;
  while (!last) {
    in.refill();
    last = in.buf & 1;
    const int type = (in.buf >> 1) & 3;
    in.drop(3);
    if (in.over()) return GAB200_PNG_TRUNCATED;
    if (type == 3) return GAB200_PNG_BLOCK_TYPE;
    if (type == 0) {
      in.drop(in.cnt & 7);   // to a byte boundary
      in.refill();
      const uint32_t len = in.peek(16), nlen = (in.buf >> 16) & 0xffff;
      in.drop(32);
      if (in.over()) return GAB200_PNG_TRUNCATED;
      if (len != (~nlen & 0xffff)) return GAB200_PNG_STORED_LENGTH;
      const int64_t at = in.pos() >> 3, avail = in.len - at, room = n - out;
      if (len > avail && avail <= room) return GAB200_PNG_TRUNCATED;   // the input ends first (or with the room)
      if (len > room) return GAB200_PNG_TOO_MUCH;
      __syncwarp();
      for (int k = lane; k < (int)len; k += 32) dst[out + k] = in.p[at + k];
      out += len;
      in.next = at + len, in.buf = 0, in.cnt = 0;
      continue;
    }
    const uint32_t* lt = sm.fixed_lit;
    const uint32_t* dt = sm.fixed_dist;
    if (type == 2) {
      const int st = dynamic_header(in, ws, lane);
      if (st != GAB200_PNG_OK) return st;
      lt = ws.lit, dt = ws.dist;
    }
    for (;;) {
      in.refill();
      int used;
      uint32_t e = lookup(lt, LIT_ROOT, in.buf, used);
      in.drop(used);
      if (in.over()) return GAB200_PNG_TRUNCATED;
      if ((e >> 24) == K_BAD) return GAB200_PNG_SYMBOL;
      const int sym = e & 0xffff;
      if (sym < 256) {
        if (out >= n) return GAB200_PNG_TOO_MUCH;
        if (lane == 0) dst[out] = (uint8_t)sym;
        out++;
        continue;
      }
      if (sym == 256) break;
      if (sym > 285) return GAB200_PNG_SYMBOL;
      const int li = sym - 257, leb = LEN_EXTRA[li];
      const int len = LEN_BASE[li] + in.peek(leb);
      in.drop(leb);
      if (in.over()) return GAB200_PNG_TRUNCATED;
      in.refill();
      e = lookup(dt, DIST_ROOT, in.buf, used);
      in.drop(used);
      if (in.over()) return GAB200_PNG_TRUNCATED;
      const int ds = e & 0xffff;
      if ((e >> 24) == K_BAD || ds > 29) return GAB200_PNG_SYMBOL;
      const int deb = DIST_EXTRA[ds];
      const int d = DIST_BASE[ds] + in.peek(deb);
      in.drop(deb);
      if (in.over()) return GAB200_PNG_TRUNCATED;
      if (d > out) return GAB200_PNG_DISTANCE;
      if (out + len > n) return GAB200_PNG_TOO_MUCH;
      __syncwarp();   // the bytes before `out`, written by any lane, are visible to every lane
      uint8_t* o = dst + out;
      if (d >= len) {
        for (int k = lane; k < len; k += 32) o[k] = o[k - d];
      } else {
        for (int k = lane; k < len; k += 32) o[k] = o[k % d - d];
      }
      out += len;
    }
  }
  if (out != n) return GAB200_PNG_TOO_LITTLE;
  in.drop(in.cnt & 7);
  in.refill();
  const uint32_t want = (uint32_t)(in.buf & 255) << 24 | (uint32_t)((in.buf >> 8) & 255) << 16 |
                        (uint32_t)((in.buf >> 16) & 255) << 8 | (uint32_t)((in.buf >> 24) & 255);
  in.drop(32);
  if (in.over()) return GAB200_PNG_TRUNCATED;
  __syncwarp();
  if (warp_adler(dst, n, lane) != want) return GAB200_PNG_ADLER;
  return GAB200_PNG_OK;
}

__host__ __device__ inline int64_t row_bytes(int W, int c) { return 1 + (int64_t)W * c; }

__global__ void __launch_bounds__(32 * PNG_DEC_WARPS) png_inflate_kernel(
    int files, int H, int W, const uint8_t* __restrict__ zdata, const int64_t* __restrict__ zoff,
    const int64_t* __restrict__ zlen, const uint8_t* __restrict__ color, uint8_t* __restrict__ scratch,
    int64_t stride, int32_t* __restrict__ status) {
  __shared__ CtaSmem sm;
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  if (wi == 0) {
    WarpSmem& ws = sm.warp[0];
    fixed_lengths(ws.lens, lane);
    build_table(ws.lens, 288, LIT_ROOT, sm.fixed_lit, 1 << LIT_ROOT, false, ws.w, lane);
    for (int s = lane; s < 32; s += 32) ws.lens[s] = 5;
    __syncwarp();
    build_table(ws.lens, 32, DIST_ROOT, sm.fixed_dist, 1 << DIST_ROOT, false, ws.w, lane);
  }
  __syncthreads();
  const int f = blockIdx.x * PNG_DEC_WARPS + wi;
  if (f >= files) return;
  const int c = color[f] == 6 ? 4 : 3;
  Bits in{zdata + zoff[f], max(zlen[f], (int64_t)0), 0, 0, 0};
  const int st = inflate_file(in, scratch + f * stride, H * row_bytes(W, c), sm, sm.warp[wi], lane);
  if (lane == 0) status[f] = st;
}

__device__ __forceinline__ uint32_t load_px(const uint8_t* p, int c) {
  uint32_t v = (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16;
  return c == 4 ? v | (uint32_t)p[3] << 24 : v;
}

// the raw pixel of filtered pixel x under filter ft, from its left (a), up (b) and up-left (cc) raw pixels
__device__ __forceinline__ uint32_t unfilter_px(int ft, uint32_t x, uint32_t a, uint32_t b, uint32_t cc) {
  if (ft == 0) return x;
  if (ft == 1) return __vadd4(x, a);
  if (ft == 2) return __vadd4(x, b);
  uint32_t r = 0;
#pragma unroll
  for (int k = 0; k < 32; k += 8) {
    const int ak = (a >> k) & 255, bk = (b >> k) & 255, ck = (cc >> k) & 255;
    int pred;
    if (ft == 3) {
      pred = (ak + bk) >> 1;
    } else {
      const int pa = abs(bk - ck), pb = abs(ak - ck), pc = abs(ak + bk - 2 * ck);
      pred = pa <= pb && pa <= pc ? ak : pb <= pc ? bk : ck;
    }
    r |= (((x >> k) + pred) & 255) << k;
  }
  return r;
}

__global__ void __launch_bounds__(32 * PNG_DEC_WARPS) png_unfilter_kernel(
    int files, int H, int W, const uint8_t* __restrict__ color, uint8_t* __restrict__ scratch, int64_t stride,
    uint8_t* __restrict__ out, int outc, int32_t* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * PNG_DEC_WARPS + (threadIdx.x >> 5);
  if (f >= files || status[f] != GAB200_PNG_OK) return;
  const int c = color[f] == 6 ? 4 : 3;
  const int64_t rs = row_bytes(W, c);
  uint8_t* buf = scratch + f * stride;
  uint8_t* img = out + (int64_t)f * H * W * outc;
  const uint32_t alpha = c == 3 ? 0xff000000u : 0u;
  const uint32_t mask = c == 4 ? 0xffffffffu : 0x00ffffffu;
  bool bad = false;
  for (int r0 = 0; r0 < H; r0 += 32) {
    const int r = r0 + lane, rows = min(32, H - r0);
    const bool row_ok = r < H;
    uint8_t* row = buf + (row_ok ? r : r0) * rs;
    const int ft = row_ok ? row[0] : 0;
    bad |= ft > 4;
    const uint8_t* above = r0 > 0 ? buf + (int64_t)(r0 - 1) * rs + 1 : nullptr;   // lane 0's row above, raw
    uint8_t* dst = img + (int64_t)r * W * outc;
    uint32_t last = 0, last2 = 0, up_prev = 0;
    for (int t = 0; t < W + rows - 1; t++) {
      const int x = t - lane;
      const bool act = row_ok && x >= 0 && x < W;
      uint32_t up = __shfl_up_sync(FULL, last, 1), ul = __shfl_up_sync(FULL, last2, 1);
      if (lane == 0) {
        const uint32_t u = act && above ? load_px(above + (int64_t)x * c, c) : 0u;
        ul = up_prev, up = u, up_prev = u;
      }
      uint32_t cur = 0;
      if (act) {
        uint8_t* px = row + 1 + (int64_t)x * c;
        cur = unfilter_px(ft, load_px(px, c), last, up, ul) & mask;
        if (outc == 4) {
          reinterpret_cast<uint32_t*>(dst)[x] = cur | alpha;
        } else {
          uint8_t* o = dst + (int64_t)x * 3;
          o[0] = cur & 255, o[1] = (cur >> 8) & 255, o[2] = (cur >> 16) & 255;
        }
        if (lane == 31)
          for (int k = 0; k < c; k++) px[k] = (cur >> (8 * k)) & 255;
      }
      last2 = last, last = cur;
    }
    __syncwarp();
  }
  if (__any_sync(FULL, bad) && lane == 0) status[f] = GAB200_PNG_FILTER;
}

}  // namespace

int64_t png_decode_stride(int H, int W) {
  if (H <= 0 || W <= 0) return -1;
  const int64_t n = (int64_t)H * (1 + 4 * (int64_t)W);   // the largest filtered stream: RGBA
  if (n > INT32_MAX) return -1;
  return (n + 255) / 256 * 256;
}

size_t png_decode_scratch_bytes(int64_t files, int H, int W) {
  const int64_t s = png_decode_stride(H, W);
  if (files <= 0 || files > INT32_MAX || s < 0) return 0;
  return (size_t)files * (size_t)s;
}

void launch_png_decode(int files, int H, int W, const uint8_t* zdata, const int64_t* zoff, const int64_t* zlen,
                       const uint8_t* color, void* scratch, uint8_t* out, int out_channels, int32_t* status,
                       cudaStream_t stream) {
  const int64_t stride = png_decode_stride(H, W);
  const int blocks = (files + PNG_DEC_WARPS - 1) / PNG_DEC_WARPS;
  uint8_t* s = static_cast<uint8_t*>(scratch);
  png_inflate_kernel<<<blocks, 32 * PNG_DEC_WARPS, 0, stream>>>(files, H, W, zdata, zoff, zlen, color, s, stride,
                                                                status);
  png_unfilter_kernel<<<blocks, 32 * PNG_DEC_WARPS, 0, stream>>>(files, H, W, color, s, stride, out, out_channels,
                                                                 status);
}

}  // namespace gab
