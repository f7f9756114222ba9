// frames.cu -- the tile-packed lossless frame store: encode once at load time, decode inside the captured iteration
// (gab200_frame_encode_plan / gab200_frame_encode / gab200_frame_decode).
//
// A frame is four uint8 planes -- R, G, B of the composited ground truth and M, its alpha bytes -- cut into 16x16
// tiles (row-major tile order, the frame's last row / column replicated past its edge).  Per tile and plane, mod 256:
//     base = v(0,0),  q = v - base,  d(y,x) = q(y,x) - q(y,x-1) - q(y-1,x) + q(y-1,x-1)   (q = 0 off the tile)
//     z = zigzag((int8) d),  b = bit length of the largest z  (0..8)
// Record (8-byte aligned): 4 bases | uint16 of the four widths (plane p in bits 4p..4p+3) | 2 zero bytes | the R, G, B,
// M payloads, 32 b bytes each: value i = 16 y + x at bits [i b, i b + b) of a little-endian bit stream.  So the 8
// values 8 l .. 8 l + 7 are exactly the b whole bytes at byte l b of the payload.  The index is `frame_base` (int64
// byte offset per frame) and `tile_off` (uint32 per (frame, tile), 8-byte units from the frame's base).
// oracle/frame_codec.py restates the format in numpy.
//
// The inverse is a 2-D inclusive prefix sum of d plus the base, and both scans parallelise over a warp: lane l owns
// row y = l / 2, columns 8 (l & 1) .. +7, i.e. values 8 l .. 8 l + 7, held as eight bytes in two words.  The row scan
// runs inside the lane (byte-wise adds) and across the lane pair; the column scan is a shuffle scan over the 16 lanes
// of one parity.
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

namespace {

constexpr int FT = 16;        // tile side
constexpr int FPLANES = 4;    // R, G, B, M
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t bytes4(uint32_t v) { return v * 0x01010101u; }   // v (< 256) in every byte

// the 8 residual bytes of one lane (bits [8 l b, 8 l b + 8 b) of the plane's payload) as two words of zigzag values
__device__ __forceinline__ void load_residuals(const uint8_t* __restrict__ payload, int b, int lane, uint32_t& lo,
                                               uint32_t& hi) {
  const int start = lane * b, w0 = start >> 3, sh = start & 7;
  const unsigned long long* P = reinterpret_cast<const unsigned long long*>(payload);   // 8-byte aligned
  unsigned long long x = __ldg(P + w0) >> (8 * sh);
  if (sh + b > 8) x |= __ldg(P + w0 + 1) << (64 - 8 * sh);
  const uint32_t m = (1u << b) - 1u;
  lo = hi = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    lo |= ((uint32_t)(x >> (j * b)) & m) << (8 * j);
    hi |= ((uint32_t)(x >> ((j + 4) * b)) & m) << (8 * j);
  }
}

// byte-wise zigzag decode: s = (z >> 1) ^ -(z & 1)
__device__ __forceinline__ uint32_t unzigzag4(uint32_t z) { return ((z >> 1) & 0x7f7f7f7fu) ^ ((z & 0x01010101u) * 0xffu); }

// Write the lane's n (<= 8) in-frame pixels v (pixel j in byte j) at dst: one 8-byte store when the row segment is
// whole and aligned, else the widest aligned stores that fit (a width like 802 leaves rows 2-byte aligned).
__device__ __forceinline__ void store_row8(uint8_t* dst, unsigned long long v, int n) {
  if (n == 8) {
    const uintptr_t a = (uintptr_t)dst;
    if ((a & 7) == 0) {
      *reinterpret_cast<unsigned long long*>(dst) = v;
    } else if ((a & 3) == 0) {
      reinterpret_cast<uint32_t*>(dst)[0] = (uint32_t)v;
      reinterpret_cast<uint32_t*>(dst)[1] = (uint32_t)(v >> 32);
    } else if ((a & 1) == 0) {
#pragma unroll
      for (int j = 0; j < 4; j++) reinterpret_cast<uint16_t*>(dst)[j] = (uint16_t)(v >> (16 * j));
    } else {
#pragma unroll
      for (int j = 0; j < 8; j++) dst[j] = (uint8_t)(v >> (8 * j));
    }
  } else {
    for (int j = 0; j < n; j++) dst[j] = (uint8_t)(v >> (8 * j));
  }
}

// One warp per (view, tile).  ids[view] selects the frame; gt (views,3,H,W) and mask (views,1,H,W, may be NULL).
__global__ void __launch_bounds__(256) frame_decode_kernel(int64_t warps, int tiles_x, int n_tiles, int H, int W,
                                                           const int32_t* __restrict__ ids,
                                                           const uint8_t* __restrict__ arena,
                                                           const int64_t* __restrict__ frame_base,
                                                           const uint32_t* __restrict__ tile_off,
                                                           uint8_t* __restrict__ gt, uint8_t* __restrict__ mask) {
  const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gw >= warps) return;
  const int lane = threadIdx.x & 31;
  const int64_t k = gw / n_tiles;
  const int t = (int)(gw - k * n_tiles);
  const int f = __ldg(ids + k);
  const uint8_t* rec = arena + __ldg(frame_base + f) + 8 * (int64_t)__ldg(tile_off + (int64_t)f * n_tiles + t);
  const uint2 h = __ldg(reinterpret_cast<const uint2*>(rec));
  const int ty = t / tiles_x, tx = t - ty * tiles_x;
  const int y = FT * ty + (lane >> 1), x0 = FT * tx + 8 * (lane & 1);
  const int n = min(8, W - x0);
  const int64_t hw = (int64_t)H * W;
  const uint8_t* payload = rec + 8;
  const int planes = mask != nullptr ? FPLANES : 3;
  for (int p = 0; p < planes; p++) {
    const int b = (h.y >> (4 * p)) & 15;
    const uint32_t base = bytes4((h.x >> (8 * p)) & 0xffu);
    uint32_t lo = base, hi = base;
    if (b != 0) {
      load_residuals(payload, b, lane, lo, hi);
      lo = unzigzag4(lo);
      hi = unzigzag4(hi);
      // row: inclusive prefix over the lane's 8 bytes, then the left half row's total on the odd lane of each pair
      lo = __vadd4(lo, lo << 8);
      lo = __vadd4(lo, lo << 16);
      hi = __vadd4(hi, hi << 8);
      hi = __vadd4(hi, hi << 16);
      hi = __vadd4(hi, bytes4(lo >> 24));
      const uint32_t left = bytes4(__shfl_up_sync(FULL, hi >> 24, 1));
      if (lane & 1) {
        lo = __vadd4(lo, left);
        hi = __vadd4(hi, left);
      }
      // column: inclusive prefix over the 16 rows (lanes of one parity)
#pragma unroll
      for (int off = 2; off < 32; off <<= 1) {
        const uint32_t ulo = __shfl_up_sync(FULL, lo, off), uhi = __shfl_up_sync(FULL, hi, off);
        if (lane >= off) {
          lo = __vadd4(lo, ulo);
          hi = __vadd4(hi, uhi);
        }
      }
      lo = __vadd4(lo, base);
      hi = __vadd4(hi, base);
      payload += 32 * b;
    }
    if (y < H && n > 0) {
      uint8_t* plane = p < 3 ? gt + (k * 3 + p) * hw : mask + k * hw;
      store_row8(plane + (int64_t)y * W + x0, (unsigned long long)lo | ((unsigned long long)hi << 32), n);
    }
  }
}

// One warp per (frame, tile), one 256-byte shared tile per warp.  PLAN: record size in 8-byte units into units[];
// else the record into arena + frame_base[f] + 8 tile_off[f, t].
template <bool PLAN>
__global__ void __launch_bounds__(128) frame_encode_kernel(int64_t warps, int tiles_x, int n_tiles, int H, int W,
                                                           const uint8_t* __restrict__ gt,
                                                           const uint8_t* __restrict__ mask, uint32_t* units,
                                                           const int64_t* __restrict__ frame_base,
                                                           const uint32_t* __restrict__ tile_off, uint8_t* arena) {
  __shared__ uint8_t tile[4][FT * FT];
  const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gw >= warps) return;
  const int lane = threadIdx.x & 31;
  uint8_t* s = tile[threadIdx.x >> 5];
  const int64_t f = gw / n_tiles;
  const int t = (int)(gw - f * n_tiles);
  const int ty = t / tiles_x, tx = t - ty * tiles_x;
  const int yl = lane >> 1, xl = 8 * (lane & 1);
  const int64_t hw = (int64_t)H * W;
  uint8_t* rec = PLAN ? nullptr : arena + frame_base[f] + 8 * (int64_t)tile_off[f * n_tiles + t];
  uint32_t bases = 0, widths = 0;
  int at = 8;   // the next payload's byte offset in the record
  for (int p = 0; p < FPLANES; p++) {
    const uint8_t* src = p < 3 ? gt + (f * 3 + p) * hw : (mask != nullptr ? mask + f * hw : nullptr);
    const int64_t row = (int64_t)min(FT * ty + yl, H - 1) * W;
    for (int j = 0; j < 8; j++)
      s[FT * yl + xl + j] = src != nullptr ? src[row + min(FT * tx + xl + j, W - 1)] : (uint8_t)255;
    __syncwarp();
    const uint8_t base = s[0];
    uint32_t zmax = 0;
    unsigned long long packed = 0;
    uint32_t z[8];
    for (int j = 0; j < 8; j++) {
      const int x = xl + j;
      auto q = [&](int yy, int xx) -> uint32_t { return yy < 0 || xx < 0 ? 0u : (uint32_t)(uint8_t)(s[FT * yy + xx] - base); };
      const uint8_t d = (uint8_t)(q(yl, x) - q(yl, x - 1) - q(yl - 1, x) + q(yl - 1, x - 1));
      const int sd = (int8_t)d;
      z[j] = (uint32_t)(((sd << 1) ^ (sd >> 7)) & 0xff);
      zmax = max(zmax, z[j]);
    }
    zmax = __reduce_max_sync(FULL, zmax);
    const int b = 32 - __clz((int)zmax);
    bases |= (uint32_t)base << (8 * p);
    widths |= (uint32_t)b << (4 * p);
    if (!PLAN && b > 0) {
      for (int j = 0; j < 8; j++) packed |= (unsigned long long)z[j] << (j * b);
      for (int j = 0; j < b; j++) rec[at + lane * b + j] = (uint8_t)(packed >> (8 * j));
    }
    at += 32 * b;
    __syncwarp();   // the tile is rewritten by the next plane
  }
  if (lane == 0) {
    if (PLAN) {
      units[gw] = (uint32_t)(at / 8);
    } else {
      *reinterpret_cast<uint2*>(rec) = make_uint2(bases, widths);
    }
  }
}

}  // namespace

int frame_tiles(int H, int W) { return ((H + FT - 1) / FT) * ((W + FT - 1) / FT); }

void launch_frame_encode_plan(int64_t frames, int H, int W, const uint8_t* gt, const uint8_t* mask, uint32_t* units,
                              cudaStream_t stream) {
  const int tiles_x = (W + FT - 1) / FT, n_tiles = frame_tiles(H, W);
  const int64_t warps = frames * n_tiles;
  if (warps == 0) return;
  frame_encode_kernel<true><<<(unsigned)((warps + 3) / 4), 128, 0, stream>>>(warps, tiles_x, n_tiles, H, W, gt, mask,
                                                                            units, nullptr, nullptr, nullptr);
  count_launch();
}

void launch_frame_encode(int64_t frames, int H, int W, const uint8_t* gt, const uint8_t* mask,
                         const int64_t* frame_base, const uint32_t* tile_off, uint8_t* arena, cudaStream_t stream) {
  const int tiles_x = (W + FT - 1) / FT, n_tiles = frame_tiles(H, W);
  const int64_t warps = frames * n_tiles;
  if (warps == 0) return;
  frame_encode_kernel<false><<<(unsigned)((warps + 3) / 4), 128, 0, stream>>>(warps, tiles_x, n_tiles, H, W, gt, mask,
                                                                             nullptr, frame_base, tile_off, arena);
  count_launch();
}

void launch_frame_decode(int views, int H, int W, const int32_t* ids, const uint8_t* arena, const int64_t* frame_base,
                         const uint32_t* tile_off, uint8_t* gt, uint8_t* mask, cudaStream_t stream) {
  const int tiles_x = (W + FT - 1) / FT, n_tiles = frame_tiles(H, W);
  const int64_t warps = (int64_t)views * n_tiles;
  if (warps == 0) return;
  frame_decode_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(warps, tiles_x, n_tiles, H, W, ids, arena,
                                                                       frame_base, tile_off, gt, mask);
  count_launch();
}

}  // namespace gab
