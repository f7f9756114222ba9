// h264.cu -- H.264 video frames encoded on the device (gab200_h264_bound / gab200_h264_scratch_bytes /
// gab200_h264_encode / gab200_h264_parameter_sets, and for streams with P pictures gab200_h264_p_bound /
// gab200_h264_state_bytes / gab200_h264_encode_stream / gab200_h264_stream_parameter_sets, and for deblocked streams
// gab200_h264_deblocked_scratch_bytes / gab200_h264_encode_deblocked, and for every option through one flags word
// gab200_h264_flags_scratch_bytes / gab200_h264_encode_flags): Constrained Baseline, CAVLC, one fixed QP,
// deblocking off (disable_deblocking_filter_idc 1) unless the stream is deblocked (idc 0, offsets 0).  An IDR
// picture's macroblocks are I_16x16 (luma and chroma modes of least SATD), I_NxN when the stream has the intra 4x4
// option (Intra_4x4 modes per 4x4 block, see h264_mb_kernel) or I_PCM; a P picture's are P_Skip, P_L0_16x16 (one
// quarter-sample vector), I_16x16, I_NxN or I_PCM.  oracle/h264.py, tests/h264_stream_oracle.py,
// tests/h264_deblock_oracle.py and tests/h264_intra4x4_oracle.py restate every step, and the tests compare their
// bytes with these.
//
// Per batch of frames the encode runs these kernels, each named for a trace:
//   h264_convert_kernel  RGB -> BT.601 limited-range Y, Cb, Cr planes padded to whole macroblocks by edge replication.
//   h264_frame_kernel    each frame's picture type and frame_num from the stream position in the state.
//   h264_mb_kernel       one launch per step of a wavefront over (frame, anti-diagonal d = mbx + mby): frame f runs
//                        diagonal step - lag f, lag 0 when every frame is an IDR picture (W/16 + H/16 - 1 launches)
//                        and LAG when a frame refers to the one before (LAG more launches per frame); a deblocked P
//                        stream runs lines d = mbx + 2 mby instead, lag LAG_DB (see LAG_DB).  One 128-thread
//                        CTA per (macroblock on d, frame): in a P picture the motion search in the previous picture;
//                        prediction from the reconstructed left / top / top-left samples of earlier diagonals (with
//                        the intra 4x4 option, <true>, also the I_NxN candidate's 16 blocks as a wavefront inside the
//                        CTA), mode decision by SATD, transform, quantisation, reconstruction into the recon planes,
//                        per-4x4 TotalCoeff, the macroblock's CAVLC bit count and the I_PCM fallback; the levels are
//                        kept for the writer.  The launch boundary is the wavefront's only synchronisation: no CTA
//                        ever waits on another.
//   h264_deblock_kernel  deblocked streams, launched after h264_mb_kernel in each step: one warp per macroblock on
//                        line mbx + 2 mby = step - lag f - DB_LAG of frame f; bS from the macroblocks' info, TotalCoeff
//                        and vectors, then the filter (8.7) of its edges from the unfiltered recon planes into the
//                        filtered planes flt, which P pictures refer to (W/16 + 2 H/16 - 2 steps per frame).
//   h264_mvp_kernel      P pictures, one thread per macroblock: the vector predictors, P_Skip and the mvd bits.
//   h264_run_kernel      P pictures, one thread per macroblock: the skip runs and their bits.
//   h264_scan_kernel     one CTA per frame: the macroblocks' bit offsets in raster order, an exclusive scan of the maps
//                        x -> x + L and x -> ceil8(x + r + 9) + 3072 (I_PCM behind a skip run of r bits, its samples
//                        byte-aligned), a family closed under composition; zeroes the slice's words and writes the
//                        slice header and the stop bit.
//   h264_write_kernel    one warp per macroblock: its bits at its offset, one lane per residual block, OR-ed into the
//                        slice's words with atomics (neighbours share the first and last word).
//   h264_ep_count_kernel one thread per 256-byte piece of the slice: for each zero-run state the piece can start in
//                        (0, 1, >= 2 zero bytes), the state it ends in and the emulation-prevention bytes it inserts.
//   h264_ep_plan_kernel  one warp per frame: the pieces' start states and output offsets in order, the sample's length
//                        and its 4-byte length prefix and NAL header.
//   h264_ep_emit_kernel  one thread per piece: its bytes, with 0x03 inserted, into the frame's output slot.
//   h264_state_kernel    the last frame's reconstruction (filtered when the stream is deblocked) and the advanced
//                        position into the stream's state.
#include <algorithm>
#include <climits>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"

namespace gab {

namespace {

constexpr int PCM_BITS = 9 + 384 * 8;        // ue(25) + the samples, before pcm_alignment_zero_bits
constexpr int MAX_LEVEL = 2063;              // what level_prefix <= 15 codes at every suffixLength
constexpr int HEADER_BITS = 22;              // the slice header (idr_pic_id 1)
constexpr int EP_PIECE = 256;                // bytes of the slice per emulation-prevention piece
constexpr int MAX_MBS = 36864;               // level 5.2's MaxFS
constexpr int BLOCKS = 27;                   // residual blocks of a macroblock, in bitstream order (see h264_mb_kernel)
constexpr int P_HEADER_BITS = 18;            // the P slice header
constexpr int SEARCH = 16;                   // integer motion search range, samples
constexpr int MVD_BITS = 2 * 17;             // se(v) of the largest |mvd|, 2 * (4 SEARCH + 3) quarter samples, twice
constexpr int INTRA_BIAS = 24;               // intra's SATD handicap against inter, in units of lambda
// I_NxN's handicap against I_16x16, in units of lambda, on top of its blocks' mode bits (see h264_mb_kernel): of the
// candidates -8, 0, 8 and 16 (scripts/video_intra4x4_sweep.py --bias), 8 gave the fewest bytes or the best Y-PSNR
// at qp 26 to 38, and at qp 20 bytes within 1.5 % of the fewest with a higher Y-PSNR than 16's.
constexpr int I4_BIAS = 8;
// A vector reaches 4 SEARCH + 3 quarter samples, and the 6-tap filter 2 samples before and 3 after: the window of a
// macroblock's reference samples spans REACH samples on each side, WIN samples in all.
constexpr int REACH = (4 * SEARCH + 3) / 4 + 3;
constexpr int WIN_OFF = REACH + 1;
constexpr int WIN = 16 + 2 * WIN_OFF;
// Frame f + 1 runs diagonal d in the launch where frame f runs d + LAG: its window reaches REACH_MB macroblocks right
// and down, so frame f must have finished diagonal d + 2 REACH_MB in an earlier launch.
constexpr int REACH_MB = (REACH + 15) / 16;
constexpr int LAG = 2 * REACH_MB + 1;
static_assert(LAG == 5, "the stream's frame lag");
static_assert(16 * REACH_MB >= REACH, "the reference window stays within REACH_MB macroblocks");
// The deblocked stream.  Filtering macroblock (x, y) changes up to 3 samples into (x - 1, y) and (x, y - 1), which
// (x + 1, y - 1)'s left edge changed before it, so the filter runs on lines x + 2 y: line t is filtered in the launch
// after the encode's own launch of the step where the encode has finished every macroblock of line t, DB_LAG steps
// behind the frame's encode line (the encode of a P stream runs on the same lines x + 2 y; an IDR-only stream keeps
// its anti-diagonals, and x + y <= x + 2 y).  Macroblock (x, y)'s filtered samples are final once (x + 1, y) and
// (x, y + 1) are filtered, line x + 2 y + 2.  Frame f + 1's window at (x, y) reaches the filtered macroblocks up to
// (x + REACH_MB, y + REACH_MB), final after line x + 2 y + 3 REACH_MB + 2 of frame f: that line must be filtered in an
// earlier step, LAG_DB > 3 REACH_MB + 2 + DB_LAG.
constexpr int DB_LAG = 0;
constexpr int LAG_DB = 3 * REACH_MB + 3 + DB_LAG;
static_assert(DB_LAG == 0 && LAG_DB == 9, "the deblocked stream's filter and frame lags");

__constant__ int8_t c_zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
__constant__ int8_t c_chroma_qp[52] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17,
                                       18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 29, 30, 31, 32, 32, 33,
                                       34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};
__constant__ int c_mf[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554},
                               {9362, 3647, 5825},  {8192, 3355, 5243},  {7282, 2893, 4559}};
__constant__ int c_v[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};
// Table 9-4, inter column: coded_block_pattern -> codeNum
__constant__ uint8_t c_inter_cbp[48] = {0,  2,  3,  7,  4,  8,  17, 13, 5,  18, 9,  14, 10, 15, 16, 11,
                                        1,  32, 33, 36, 34, 37, 44, 40, 35, 45, 38, 41, 39, 42, 43, 19,
                                        6,  24, 25, 20, 26, 21, 46, 28, 27, 47, 22, 29, 23, 30, 31, 12};
// Table 9-4, intra column: coded_block_pattern -> codeNum
__constant__ uint8_t c_intra_cbp[48] = {3,  29, 30, 17, 31, 18, 37, 8,  32, 38, 19, 9,  20, 10, 11, 2,
                                        16, 33, 34, 21, 35, 22, 39, 4,  36, 40, 23, 5,  24, 6,  7,  1,
                                        41, 42, 43, 25, 44, 26, 46, 12, 45, 47, 27, 13, 28, 14, 15, 0};
// luma4x4BlkIdx -> (x, y) of the 4x4 block in the macroblock, in blocks
__constant__ int8_t c_blk_x[16] = {0, 1, 0, 1, 2, 3, 2, 3, 0, 1, 0, 1, 2, 3, 2, 3};
__constant__ int8_t c_blk_y[16] = {0, 0, 1, 1, 0, 0, 1, 1, 2, 2, 3, 3, 2, 2, 3, 3};

// Table 9-5, [TrailingOnes + 4 TotalCoeff]
__constant__ uint8_t c_ct_len[4][68] = {
    {1,  0,  0,  0,  6,  2,  0,  0,  8,  6,  3,  0,  9,  8,  7,  5,  10, 9,  8,  6,  11, 10, 9,
     7,  13, 11, 10, 8,  13, 13, 11, 9,  13, 13, 13, 10, 14, 14, 13, 11, 14, 14, 14, 13, 15, 15,
     14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16},
    {2,  0,  0,  0,  6,  2,  0,  0,  6,  5,  3,  0,  7,  6,  6,  4,  8,  6,  6,  4,  8,  7,  7,
     5,  9,  8,  8,  6,  11, 9,  9,  6,  11, 11, 11, 7,  12, 11, 11, 9,  12, 12, 12, 11, 12, 12,
     12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14},
    {4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4,  7,  5,  5,  4,  7,  5,  5,  4,  7,  6,  6,  4,  7,  6,  6,  4,  8,  7,
     7, 5, 8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10},
    {6, 0, 0, 0, 6, 6, 0, 0, 6, 6, 6, 0, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6,
     6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6}};
__constant__ uint8_t c_ct_code[4][68] = {
    {1,  0,  0, 0,  5, 1, 0, 0,  7,  4,  1, 0,  7,  6,  5,  3,  7,  6,  5,  3, 7, 6, 5,
     4,  15, 6, 5,  4, 11, 14, 5, 4, 8, 10, 13, 4, 15, 14, 9, 4, 11, 10, 13, 12, 15, 14,
     9,  12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8},
    {3,  0,  0,  0,  11, 2,  0,  0,  7,  7,  3,  0,  7,  10, 9,  5,  7,  6, 5, 4, 4, 6, 5,
     6,  7,  6,  5,  8,  15, 6,  5,  4,  11, 14, 13, 4,  15, 10, 9,  4,  11, 14, 13, 12, 8, 10,
     9,  8,  15, 14, 13, 12, 11, 10, 9,  12, 7,  11, 6,  8,  9,  8,  10, 1,  7,  6,  5,  4},
    {15, 0,  0,  0,  15, 14, 0,  0,  11, 15, 13, 0,  8,  12, 14, 12, 15, 10, 11, 11, 11, 8, 9,
     10, 9,  14, 13, 9,  8,  10, 9,  8,  15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14,
     9,  12, 8,  10, 13, 8,  13, 7,  9,  12, 9,  12, 11, 10, 5,  8,  7,  6,  1,  4,  3,  2},
    {3,  0,  0,  0,  0,  1,  0,  0,  4,  5,  6,  0,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18,
     19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41,
     42, 43, 44, 45, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 59, 60, 61, 62, 63}};
__constant__ uint8_t c_cdc_len[20] = {2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7};
__constant__ uint8_t c_cdc_code[20] = {1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0};
// Tables 9-7 / 9-8, [TotalCoeff - 1][total_zeros]
__constant__ uint8_t c_tz_len[15][16] = {
    {1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9}, {3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6},
    {4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6},       {5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5},
    {4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5},             {6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6},
    {6, 5, 3, 3, 3, 2, 3, 4, 3, 6},                   {6, 4, 5, 3, 2, 2, 3, 3, 6},
    {6, 6, 4, 2, 2, 3, 2, 5},                         {5, 5, 3, 2, 2, 2, 4},
    {4, 4, 3, 3, 1, 3},                               {4, 4, 2, 1, 3},
    {3, 3, 1, 2},                                     {2, 2, 1},
    {1, 1}};
__constant__ uint8_t c_tz_code[15][16] = {
    {1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1}, {7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0},
    {5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0},       {3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0},
    {5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0},             {1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0},
    {1, 1, 5, 4, 3, 3, 2, 1, 1, 0},                   {1, 1, 1, 3, 3, 2, 2, 1, 0},
    {1, 0, 1, 3, 2, 1, 1, 1},                         {1, 0, 1, 3, 2, 1, 1},
    {0, 1, 1, 2, 1, 3},                               {0, 1, 1, 1, 1},
    {0, 1, 1, 1},                                     {0, 1, 1},
    {0, 1}};
__constant__ uint8_t c_ctz_len[3][4] = {{1, 2, 3, 3}, {1, 2, 2}, {1, 1}};
__constant__ uint8_t c_ctz_code[3][4] = {{1, 1, 1, 0}, {1, 1, 0}, {1, 0}};
// Table 9-10, [min(zerosLeft, 7) - 1][run_before]
__constant__ uint8_t c_rb_len[7][15] = {{1, 1},          {1, 2, 2},          {2, 2, 2, 2},         {2, 2, 2, 3, 3},
                                        {2, 2, 3, 3, 3, 3}, {2, 3, 3, 3, 3, 3, 3}, {3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
__constant__ uint8_t c_rb_code[7][15] = {{1, 0},          {1, 1, 0},          {3, 2, 1, 0},         {3, 2, 1, 1, 0},
                                         {3, 2, 3, 2, 1, 0}, {3, 0, 1, 3, 2, 5, 4}, {7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1}};

// The per-frame scratch: offsets from the frame's base (each 256-byte aligned), and the frame stride.
struct Layout {
  int W, H, wm, hm, nmb, pieces, deblock;
  // flt: the picture a P picture refers to and the state keeps -- the deblocked copy of rec, or rec itself;
  // modes: the I_NxN streams' Intra4x4PredMode per 4x4 block, 8 bytes per macroblock
  int64_t src, rec, tot, lev, info, bits, off, mv, mvd, run, raw, ep, meta, flt, modes, stride;
};

int64_t align256(int64_t x) { return (x + 255) / 256 * 256; }

int64_t raw_bytes_bound(int nmb) { return (HEADER_BITS + (int64_t)nmb * (PCM_BITS + 7) + 1 + 7) / 8; }
// A P slice: a skip run of at most 3 bits per macroblock it closes, the mvd and I_PCM at its worst alignment.
int64_t raw_bytes_bound_p(int nmb) {
  return (P_HEADER_BITS + (int64_t)nmb * (3 + MVD_BITS + PCM_BITS + 7) + 1 + 7) / 8;
}

Layout layout(int H, int W, bool deblock = false, bool intra4x4 = false) {
  Layout l;
  l.deblock = deblock;
  l.W = W;
  l.H = H;
  l.wm = (W + 15) / 16;
  l.hm = (H + 15) / 16;
  l.nmb = l.wm * l.hm;
  const int64_t raw = std::max(raw_bytes_bound(l.nmb), raw_bytes_bound_p(l.nmb));
  l.pieces = (int)((raw + EP_PIECE - 1) / EP_PIECE);
  const int64_t plane = (int64_t)l.nmb * 384;   // Y, Cb, Cr of every macroblock
  int64_t o = 0;
  l.src = o;  o = align256(o + plane);
  l.rec = o;  o = align256(o + plane);
  l.tot = o;  o = align256(o + (int64_t)l.nmb * 24);                 // TotalCoeff: 16 luma, 4 Cb, 4 Cr per macroblock
  l.lev = o;  o = align256(o + (int64_t)l.nmb * BLOCKS * 16 * 2);    // int16 levels in scan order
  l.info = o; o = align256(o + (int64_t)l.nmb * 4);
  l.bits = o; o = align256(o + (int64_t)l.nmb * 4);
  l.off = o;  o = align256(o + (int64_t)l.nmb * 4);
  l.mv = o;   o = align256(o + (int64_t)l.nmb * 4);                   // P: x | y << 16, quarter samples
  l.mvd = o;  o = align256(o + (int64_t)l.nmb * 4);
  l.run = o;  o = align256(o + (int64_t)l.nmb * 4);                   // P: the skip run coded before the macroblock
  l.raw = o;  o = align256(o + (raw + 7) / 4 * 4 + 4);                // the slice's words, one spare
  l.ep = o;   o = align256(o + (int64_t)l.pieces * 16);               // per piece: 3 counts + end states | start state
  l.meta = o; o = align256(o + 16);                                   // raw byte count, P picture, frame_num
  l.flt = l.rec;
  if (deblock) { l.flt = o; o = align256(o + plane); }                 // the deblocked picture
  l.modes = 0;
  if (intra4x4) { l.modes = o; o = align256(o + (int64_t)l.nmb * 8); } // raster 4x4 block k in bits 4k .. 4k + 3
  l.stride = o;
  return l;
}

__device__ __forceinline__ int clip255(int v) { return min(max(v, 0), 255); }

// Plane layout: luma rows of 16 wm bytes, then Cb and Cr rows of 8 wm bytes.
struct Planes {
  uint8_t* y;
  uint8_t* cb;
  uint8_t* cr;
  int ys, cs;   // row strides
  __device__ Planes(uint8_t* base, const Layout& l) {
    ys = 16 * l.wm;
    cs = 8 * l.wm;
    y = base;
    cb = base + (int64_t)ys * 16 * l.hm;
    cr = cb + (int64_t)cs * 8 * l.hm;
  }
  __device__ uint8_t* chroma(int p) const { return p ? cr : cb; }
};

// ---- colour conversion -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) h264_convert_kernel(const uint8_t* __restrict__ rgb, uint8_t* scratch,
                                                            Layout l) {
  const int f = blockIdx.y;
  const int cw = 8 * l.wm, chh = 8 * l.hm;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cw * chh) return;
  const int cx = i % cw, cy = i / cw;
  const uint8_t* img = rgb + (int64_t)f * l.H * l.W * 3;
  Planes p(scratch + (int64_t)f * l.stride + l.src, l);
  for (int dy = 0; dy < 2; dy++)
    for (int dx = 0; dx < 2; dx++) {
      const int x = min(2 * cx + dx, l.W - 1), y = min(2 * cy + dy, l.H - 1);
      const uint8_t* px = img + ((int64_t)y * l.W + x) * 3;
      p.y[(2 * cy + dy) * p.ys + 2 * cx + dx] = (uint8_t)(((66 * px[0] + 129 * px[1] + 25 * px[2] + 128) >> 8) + 16);
    }
  const int sx = 2 * min(cx, l.W / 2 - 1), sy = 2 * min(cy, l.H / 2 - 1);
  int r4 = 0, g4 = 0, b4 = 0;
  for (int dy = 0; dy < 2; dy++)
    for (int dx = 0; dx < 2; dx++) {
      const uint8_t* px = img + ((int64_t)(sy + dy) * l.W + sx + dx) * 3;
      r4 += px[0];
      g4 += px[1];
      b4 += px[2];
    }
  p.cb[cy * p.cs + cx] = (uint8_t)(((-38 * r4 - 74 * g4 + 112 * b4 + 512) >> 10) + 128);
  p.cr[cy * p.cs + cx] = (uint8_t)(((112 * r4 - 94 * g4 - 18 * b4 + 512) >> 10) + 128);
}

// ---- bits ------------------------------------------------------------------------------------------------------
// OR `len` (<= 32) bits of `code` into the big-endian bit string held in little-endian words, at bit `pos`.
__device__ __forceinline__ void put_bits(uint32_t* buf, uint32_t pos, uint32_t code, int len) {
  if (len <= 0) return;
  const uint64_t v = (uint64_t)code << (64 - len - (int)(pos & 31));
  const uint32_t hi = (uint32_t)(v >> 32), lo = (uint32_t)v;
  if (hi) atomicOr(buf + (pos >> 5), __byte_perm(hi, 0, 0x0123));
  if (lo) atomicOr(buf + (pos >> 5) + 1, __byte_perm(lo, 0, 0x0123));
}

__device__ __forceinline__ int ue_bits(int v) { return 2 * (32 - __clz(v + 1)) - 1; }

struct BitSink {
  uint32_t* buf;
  uint32_t pos;
  int n;
  __device__ void u(uint32_t code, int len) {
    if (buf) put_bits(buf, pos + n, code, len);
    n += len;
  }
};

// One residual_block_cavlc (9.2) of coefficients c[0 .. maxn) in scan order, context nc (-1: chroma DC); returns bits.
__device__ __forceinline__ int cavlc_block(const int* c, int maxn, int nc, BitSink& s) {
  const int n0 = s.n;
  int total = 0, last = -1;
  for (int i = 0; i < maxn; i++)
    if (c[i]) {
      total++;
      last = i;
    }
  int t1 = 0;
  for (int i = last; i >= 0 && t1 < 3; i--) {
    if (!c[i]) continue;
    if (c[i] == 1 || c[i] == -1) t1++;
    else break;
  }
  if (nc < 0) {
    s.u(c_cdc_code[4 * total + t1], c_cdc_len[4 * total + t1]);
  } else {
    const int tab = nc < 2 ? 0 : nc < 4 ? 1 : nc < 8 ? 2 : 3;
    s.u(c_ct_code[tab][4 * total + t1], c_ct_len[tab][4 * total + t1]);
  }
  if (total == 0) return s.n - n0;
  int sl = (total > 10 && t1 < 3) ? 1 : 0;
  int k = 0;   // nonzero coefficients seen, highest frequency first
  for (int i = last; i >= 0; i--) {
    const int v = c[i];
    if (!v) continue;
    if (k < t1) {
      s.u(v < 0, 1);
    } else {
      int code = v > 0 ? 2 * v - 2 : -2 * v - 1;
      if (k == t1 && t1 < 3) code -= 2;
      int prefix, suffix, slen;
      if (sl == 0) {
        if (code < 14) { prefix = code; suffix = 0; slen = 0; }
        else if (code < 30) { prefix = 14; suffix = code - 14; slen = 4; }
        else { prefix = 15; suffix = code - 30; slen = 12; }
      } else if (code < (15 << sl)) {
        prefix = code >> sl; suffix = code & ((1 << sl) - 1); slen = sl;
      } else {
        prefix = 15; suffix = code - (15 << sl); slen = 12;
      }
      s.u(1, prefix + 1);
      s.u((uint32_t)suffix, slen);
      if (sl == 0) sl = 1;
      if (abs(v) > (3 << (sl - 1)) && sl < 6) sl++;
    }
    k++;
  }
  const int zeros = last + 1 - total;
  if (total < maxn) {
    if (nc < 0) s.u(c_ctz_code[total - 1][zeros], c_ctz_len[total - 1][zeros]);
    else s.u(c_tz_code[total - 1][zeros], c_tz_len[total - 1][zeros]);
  }
  int left = zeros, prev = last;
  for (int i = last - 1; i >= 0 && left > 0; i--) {
    if (!c[i]) continue;
    const int run = prev - i - 1, t = min(left, 7) - 1;
    s.u(c_rb_code[t][run], c_rb_len[t][run]);
    left -= run;
    prev = i;
  }
  return s.n - n0;
}

// TotalCoeff grid of a frame: per macroblock 16 luma (luma4x4BlkIdx raster: [by * 4 + bx]), 4 Cb, 4 Cr.
__device__ __forceinline__ int tot_at(const uint8_t* tot, const Layout& l, int plane, int x, int y) {
  const int per = plane == 0 ? 4 : 2;
  const int mb = (y / per) * l.wm + x / per;
  const int bx = x % per, by = y % per;
  return tot[(int64_t)mb * 24 + (plane == 0 ? by * 4 + bx : 16 + 4 * (plane - 1) + by * 2 + bx)];
}

__device__ int nc_of(const uint8_t* tot, const Layout& l, int plane, int x, int y) {
  const int a = x > 0 ? tot_at(tot, l, plane, x - 1, y) : -1;
  const int b = y > 0 ? tot_at(tot, l, plane, x, y - 1) : -1;
  if (a >= 0 && b >= 0) return (a + b + 1) >> 1;
  return a >= 0 ? a : b >= 0 ? b : 0;
}

// Block id (0 .. 26, bitstream order) -> (plane, x, y of its 4x4 block in the plane's grid, max coefficients).
__device__ void block_geom(int id, int mx, int my, int& plane, int& x, int& y, int& maxn) {
  if (id == 0) { plane = 0; x = 4 * mx; y = 4 * my; maxn = 16; }
  else if (id <= 16) { plane = 0; x = 4 * mx + c_blk_x[id - 1]; y = 4 * my + c_blk_y[id - 1]; maxn = 15; }
  else if (id <= 18) { plane = -1; x = y = 0; maxn = 4; }
  else { const int b = (id - 19) & 3; plane = 1 + (id - 19) / 4; x = 2 * mx + (b & 1); y = 2 * my + (b >> 1); maxn = 15; }
}

// A macroblock's info word: luma mode (bits 0-1), chroma mode (2-3), CodedBlockPatternChroma (4-5), I_16x16 AC
// coded (6), I_PCM (7), P_L0_16x16 (8), its CodedBlockPatternLuma (9-12), P_Skip (13), I_NxN (14, with its
// CodedBlockPatternLuma in 9-12 and its luma blocks coded as an inter macroblock's: 16 coefficients, no DC block).
__device__ __forceinline__ bool block_present(int id, int info) {
  const bool inter = info & (1 << 8 | 1 << 14);
  const int cbpc = (info >> 4) & 3;
  if (id == 0) return !inter;
  if (id <= 16) return inter ? (info >> (9 + ((id - 1) >> 2))) & 1 : (info >> 6) & 1;
  return id <= 18 ? cbpc >= 1 : cbpc == 2;
}

__device__ __forceinline__ int i16_mb_type(int info, bool is_p) {
  return 1 + (info & 3) + 4 * ((info >> 4) & 3) + ((info >> 6) & 1 ? 12 : 0) + (is_p ? 5 : 0);
}

__device__ __forceinline__ int inter_cbp(int info) { return ((info >> 9) & 15) | ((info >> 4) & 3) << 4; }

// mb_type through mb_qp_delta: I_16x16 (mb_type + 5 in a P slice), or P_L0_16x16 without its mvd
__device__ __forceinline__ int mb_header_bits(int info, bool is_p) {
  if ((info >> 8) & 1) return 1 + ue_bits(c_inter_cbp[inter_cbp(info)]) + (inter_cbp(info) ? 1 : 0);
  return ue_bits(i16_mb_type(info, is_p)) + ue_bits((info >> 2) & 3) + 1;
}

// ---- Intra_4x4 (8.3.1) -------------------------------------------------------------------------------------------
// luma4x4BlkIdx of the 4x4 block at (bx, by) of a macroblock
__device__ __forceinline__ int blk_idx(int bx, int by) { return 8 * (by >> 1) + 4 * (bx >> 1) + 2 * (by & 1) + (bx & 1); }

__device__ __forceinline__ int mode_at(uint64_t modes, int bx, int by) { return (int)(modes >> (4 * (4 * by + bx))) & 15; }

// 8.3.1.1: predIntra4x4PredMode of block (bx, by) of macroblock (mx, my), whose own modes are `own`; a neighbouring
// macroblock that is unavailable gives 2, one that is not I_NxN gives mode 2 for its blocks.
__device__ __forceinline__ int i4_pred_mode(uint64_t own, const int* info, const uint64_t* modes, int wm, int mx,
                                            int my, int bx, int by) {
  int a, b;
  if (bx > 0) a = mode_at(own, bx - 1, by);
  else if (mx == 0) return 2;
  else a = (info[my * wm + mx - 1] >> 14) & 1 ? mode_at(modes[my * wm + mx - 1], 3, by) : 2;
  if (by > 0) b = mode_at(own, bx, by - 1);
  else if (my == 0) return 2;
  else b = (info[(my - 1) * wm + mx] >> 14) & 1 ? mode_at(modes[(my - 1) * wm + mx], bx, 3) : 2;
  return min(a, b);
}

// An I_NxN macroblock's mb_type through mb_qp_delta: ue(0) (ue(5) in a P slice), per block in luma4x4BlkIdx order
// prev_intra4x4_pred_mode_flag or 0 and rem_intra4x4_pred_mode u(3), intra_chroma_pred_mode, coded_block_pattern
// (intra column), mb_qp_delta; returns its bits, writes them when s has a buffer.
__device__ int i4_header(const int* info, const uint64_t* modes, int wm, int mx, int my, bool is_p, BitSink& s) {
  const int n0 = s.n, me = info[my * wm + mx];
  const uint64_t own = modes[my * wm + mx];
  s.u(is_p ? 6 : 1, is_p ? 5 : 1);
  for (int k = 0; k < 16; k++) {
    const int bx = c_blk_x[k], by = c_blk_y[k];
    const int m = mode_at(own, bx, by), pm = i4_pred_mode(own, info, modes, wm, mx, my, bx, by);
    if (m == pm) s.u(1, 1);
    else s.u(m < pm ? m : m - 1, 4);
  }
  const int cmode = (me >> 2) & 3, cbp = ((me >> 9) & 15) | ((me >> 4) & 3) << 4, code = c_intra_cbp[cbp];
  s.u(cmode + 1, ue_bits(cmode));
  s.u(code + 1, ue_bits(code));
  if (cbp) s.u(1, 1);                            // mb_qp_delta 0
  return s.n - n0;
}

// 8.3.1.2: the prediction of Intra4x4PredMode `mode` at (x, y) of a 4x4 block from its edge e: e[3 - j] = p[-1, j],
// e[4] = p[-1, -1], e[5 + i] = p[i, -1] (i = 0 .. 7, p[4..7, -1] already substituted when unavailable); dc is mode 2's.
__device__ __forceinline__ int pred4(const int* e, int mode, int dc, int x, int y) {
  auto P = [&](int i, int j) { return j < 0 ? e[5 + i] : e[3 - j]; };   // p[i, j], i = -1 or j = -1
  auto f3 = [](int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; };
  auto f2 = [](int a, int b) { return (a + b + 1) >> 1; };
  switch (mode) {
    case 0: return P(x, -1);
    case 1: return P(-1, y);
    case 2: return dc;
    case 3: return x == 3 && y == 3 ? (P(6, -1) + 3 * P(7, -1) + 2) >> 2 : f3(P(x + y, -1), P(x + y + 1, -1), P(x + y + 2, -1));
    case 4:
      if (x > y) return f3(P(x - y - 2, -1), P(x - y - 1, -1), P(x - y, -1));
      if (x < y) return f3(P(-1, y - x - 2), P(-1, y - x - 1), P(-1, y - x));
      return f3(P(0, -1), P(-1, -1), P(-1, 0));
    case 5: {
      const int z = 2 * x - y;
      if (z >= 0 && !(z & 1)) return f2(P(x - (y >> 1) - 1, -1), P(x - (y >> 1), -1));
      if (z > 0) return f3(P(x - (y >> 1) - 2, -1), P(x - (y >> 1) - 1, -1), P(x - (y >> 1), -1));
      if (z == -1) return f3(P(-1, 0), P(-1, -1), P(0, -1));
      return f3(P(-1, y - 1), P(-1, y - 2), P(-1, y - 3));
    }
    case 6: {
      const int z = 2 * y - x;
      if (z >= 0 && !(z & 1)) return f2(P(-1, y - (x >> 1) - 1), P(-1, y - (x >> 1)));
      if (z > 0) return f3(P(-1, y - (x >> 1) - 2), P(-1, y - (x >> 1) - 1), P(-1, y - (x >> 1)));
      if (z == -1) return f3(P(-1, 0), P(-1, -1), P(0, -1));
      return f3(P(x - 1, -1), P(x - 2, -1), P(x - 3, -1));
    }
    case 7:
      if (!(y & 1)) return f2(P(x + (y >> 1), -1), P(x + (y >> 1) + 1, -1));
      return f3(P(x + (y >> 1), -1), P(x + (y >> 1) + 1, -1), P(x + (y >> 1) + 2, -1));
    default: {
      const int z = x + 2 * y;
      if (z > 5) return P(-1, 3);
      if (z == 5) return (P(-1, 2) + 3 * P(-1, 3) + 2) >> 2;
      if (!(z & 1)) return f2(P(-1, y + (x >> 1)), P(-1, y + (x >> 1) + 1));
      return f3(P(-1, y + (x >> 1)), P(-1, y + (x >> 1) + 1), P(-1, y + (x >> 1) + 2));
    }
  }
}

// ---- the macroblock kernel ---------------------------------------------------------------------------------------
__device__ __forceinline__ int quant(int c, int mf, int qbits, int f) {
  const int q = (abs(c) * mf + f) >> qbits;
  return c < 0 ? -q : q;
}

__device__ __forceinline__ int pos_class(int i) {   // raster index in a 4x4 block -> 0 (even, even), 1 (odd, odd), 2
  const int r = i >> 2, c = i & 3;
  return (!(r & 1) && !(c & 1)) ? 0 : ((r & 1) && (c & 1)) ? 1 : 2;
}

// 8.5.12.2 on a 4x4 block d (raster, row-major), in place -> residual (h + 32) >> 6
__device__ void idct4(int* d) {
  for (int i = 0; i < 4; i++) {
    int* r = d + 4 * i;
    const int e0 = r[0] + r[2], e1 = r[0] - r[2], e2 = (r[1] >> 1) - r[3], e3 = r[1] + (r[3] >> 1);
    r[0] = e0 + e3; r[1] = e1 + e2; r[2] = e1 - e2; r[3] = e0 - e3;
  }
  for (int j = 0; j < 4; j++) {
    const int f0 = d[j], f1 = d[4 + j], f2 = d[8 + j], f3 = d[12 + j];
    const int g0 = f0 + f2, g1 = f0 - f2, g2 = (f1 >> 1) - f3, g3 = f1 + (f3 >> 1);
    d[j] = (g0 + g3 + 32) >> 6; d[4 + j] = (g1 + g2 + 32) >> 6; d[8 + j] = (g1 - g2 + 32) >> 6;
    d[12 + j] = (g0 - g3 + 32) >> 6;
  }
}

struct MbShared {
  int src[384];          // Y (16x16), Cb (8x8), Cr (8x8)
  int pred[384];         // the chosen modes' predictions
  int ipred[384];        // P: the inter prediction at the chosen vector
  int top[32], left[32]; // luma 0..15, Cb 16..23, Cr 24..31
  int tl[3];
  int par[3][8];         // per plane: DC value(s) and the plane parameters a, b, c
  int cost[8];           // SATD of luma modes 0..3, chroma modes 0..3
  int w[24][16];         // transform coefficients, then dequantised coefficients
  int lev[24][16];       // quantised levels (raster; [0] unused in intra blocks)
  int dc[16], cdc[2][4]; // quantised DC levels (luma [by * 4 + bx], chroma raster)
  int dcr[16], cdcr[2][4];
  int tot[24];
  int c9[9];             // P: the costs of a refinement's candidates
  uint8_t win[WIN * WIN];// P: the reference samples around the macroblock, coordinates clamped to the picture
  int maxlev, bits, lmode, cmode, cbpl, cbpc, pcm, inter, key, mvx, mvy, icost;
};

// The I_NxN candidate's part (h264_mb_kernel<true> only); its levels and TotalCoeff go to lev[0..15] / tot[0..15].
struct MbSharedI4 : MbShared {
  int r4[256];           // the reconstruction, raster
  int c4[2][9];          // SATD of the current step's (block, mode) pairs
  uint64_t own;          // the chosen modes, raster block k in bits 4k .. 4k + 3
  int sum4, mbits4, max4, nxn;   // sum of the blocks' costs, their mode bits, the largest |level|, I_NxN chosen
};

__device__ int predict(const MbShared& s, int plane, int mode, int x, int y) {
  if (plane == 0) {
    switch (mode) {
      case 0: return s.top[x];
      case 1: return s.left[y];
      case 2: return s.par[0][0];
      default: return clip255((s.par[0][1] + s.par[0][2] * (x - 7) + s.par[0][3] * (y - 7) + 16) >> 5);
    }
  }
  const int o = 16 + 8 * (plane - 1);
  switch (mode) {
    case 0: return s.par[plane][(y >> 2) * 2 + (x >> 2)];
    case 1: return s.left[o + y];
    case 2: return s.top[o + x];
    default: return clip255((s.par[plane][4] + s.par[plane][5] * (x - 3) + s.par[plane][6] * (y - 3) + 16) >> 5);
  }
}

__device__ __forceinline__ int se_bits(int v) { return ue_bits(v > 0 ? 2 * v - 1 : -2 * v); }
__device__ __forceinline__ int lambda_of(int qp) { return 1 << max(0, (qp - 12) / 6); }

__device__ __forceinline__ int tap6(const uint8_t* p, int step) {
  return p[-2 * step] - 5 * p[-step] + 20 * p[0] + 20 * p[step] - 5 * p[2 * step] + p[3 * step];
}

// 8.4.2.2.1: the luma sample at (x, y) of the macroblock displaced by (mvx, mvy) quarter samples, from the window.
__device__ __forceinline__ int luma_at(const uint8_t* win, int x, int y, int mvx, int mvy) {
  const int xf = mvx & 3, yf = mvy & 3;
  const uint8_t* g = win + (WIN_OFF + y + (mvy >> 2)) * WIN + WIN_OFF + x + (mvx >> 2);
  if (!xf && !yf) return g[0];
  const int b = clip255((tap6(g, 1) + 16) >> 5), h = clip255((tap6(g, WIN) + 16) >> 5);
  const int s = clip255((tap6(g + WIN, 1) + 16) >> 5), m = clip255((tap6(g + 1, WIN) + 16) >> 5);
  int j = 0;
  if ((xf == 2 && yf) || (yf == 2 && xf)) {
    int v[6];
    for (int k = 0; k < 6; k++) v[k] = tap6(g + k - 2, WIN);
    j = clip255((v[0] - 5 * v[1] + 20 * v[2] + 20 * v[3] - 5 * v[4] + v[5] + 512) >> 10);
  }
  auto avg = [](int p, int q) { return (p + q + 1) >> 1; };
  switch (yf * 4 + xf) {
    case 1: return avg(g[0], b);
    case 2: return b;
    case 3: return avg(g[1], b);
    case 4: return avg(g[0], h);
    case 5: return avg(b, h);
    case 6: return avg(b, j);
    case 7: return avg(b, m);
    case 8: return h;
    case 9: return avg(h, j);
    case 10: return j;
    case 11: return avg(j, m);
    case 12: return avg(g[WIN], h);
    case 13: return avg(h, s);
    case 14: return avg(j, s);
    default: return avg(m, s);
  }
}

// 8.4.2.2.2: the chroma sample at (x, y) of plane p's coded picture displaced by (mvx, mvy) eighth samples.
__device__ __forceinline__ int chroma_at(const Planes& ref, const Layout& l, int p, int x, int y, int mvx, int mvy) {
  const int xi = x + (mvx >> 3), yi = y + (mvy >> 3), xf = mvx & 7, yf = mvy & 7;
  const int w1 = 8 * l.wm - 1, h1 = 8 * l.hm - 1;
  const uint8_t* pl = ref.chroma(p);
  const int x0 = min(max(xi, 0), w1), x1 = min(max(xi + 1, 0), w1);
  const int y0 = min(max(yi, 0), h1) * ref.cs, y1 = min(max(yi + 1, 0), h1) * ref.cs;
  return ((8 - xf) * (8 - yf) * pl[y0 + x0] + xf * (8 - yf) * pl[y0 + x1] + (8 - xf) * yf * pl[y1 + x0] +
          xf * yf * pl[y1 + x1] + 32) >> 6;
}

__device__ __forceinline__ int satd4(const int* r) {   // r: 16 residuals, raster; sum of |4x4 Hadamard|
  int q[16];
  for (int i = 0; i < 4; i++) {
    const int a0 = r[4 * i] + r[4 * i + 1], a1 = r[4 * i] - r[4 * i + 1];
    const int a2 = r[4 * i + 2] + r[4 * i + 3], a3 = r[4 * i + 2] - r[4 * i + 3];
    q[4 * i] = a0 + a2; q[4 * i + 1] = a1 + a3; q[4 * i + 2] = a0 - a2; q[4 * i + 3] = a1 - a3;
  }
  int sum = 0;
  for (int j = 0; j < 4; j++) {
    const int a0 = q[j] + q[4 + j], a1 = q[j] - q[4 + j], a2 = q[8 + j] + q[12 + j], a3 = q[8 + j] - q[12 + j];
    sum += abs(a0 + a2) + abs(a1 + a3) + abs(a0 - a2) + abs(a1 - a3);
  }
  return sum;
}

__constant__ int8_t c_nb[8][2] = {{-1, -1}, {0, -1}, {1, -1}, {-1, 0}, {1, 0}, {-1, 1}, {0, 1}, {1, 1}};  // (dx, dy)

// The motion search of a P macroblock (128 threads): an integer full search over +-SEARCH samples by SAD, then a
// half- and a quarter-sample refinement over the 8 neighbours by SATD, each cost + lambda * the vector's se(v) bits;
// every minimum keeps the first candidate (raster order, then the centre before its neighbours).  Leaves the vector in
// s.mvx / s.mvy, its cost in s.icost and its luma and chroma prediction in s.ipred.
__device__ __forceinline__ void motion_search(MbShared& s, const Planes& ref, const Layout& l, int mx, int my, int qp) {
  const int t = threadIdx.x, L = lambda_of(qp);
  const int x0 = 16 * mx - WIN_OFF, y0 = 16 * my - WIN_OFF, wc = 16 * l.wm, hc = 16 * l.hm;
  for (int i = t; i < WIN * WIN; i += 128) {
    const int x = min(max(x0 + i % WIN, 0), wc - 1), y = min(max(y0 + i / WIN, 0), hc - 1);
    s.win[i] = ref.y[(int64_t)y * ref.ys + x];
  }
  if (t == 0) s.key = INT_MAX;
  __syncthreads();
  constexpr int SIDE = 2 * SEARCH + 1;
  int best = INT_MAX;
  for (int c = t; c < SIDE * SIDE; c += 128) {
    const int dx = c % SIDE - SEARCH, dy = c / SIDE - SEARCH;
    int sad = 0;
    for (int y = 0; y < 16; y++) {
      const uint8_t* row = s.win + (WIN_OFF + y + dy) * WIN + WIN_OFF + dx;
      for (int x = 0; x < 16; x++) sad += abs(s.src[16 * y + x] - (int)row[x]);
    }
    best = min(best, (sad + L * (se_bits(4 * dx) + se_bits(4 * dy))) << 11 | c);
  }
  atomicMin(&s.key, best);
  __syncthreads();
  int mvx = 4 * ((s.key & 2047) % SIDE - SEARCH), mvy = 4 * ((s.key & 2047) / SIDE - SEARCH);
  for (int step = 2; step >= 1; step--) {
    if (t < 9) {
      const int vx = mvx + (t ? c_nb[t - 1][0] * step : 0), vy = mvy + (t ? c_nb[t - 1][1] * step : 0);
      s.c9[t] = L * (se_bits(vx) + se_bits(vy));
    }
    __syncthreads();
    for (int task = t; task < 9 * 16; task += 128) {
      const int k = task / 16, bx = task & 3, by = (task >> 2) & 3;
      const int vx = mvx + (k ? c_nb[k - 1][0] * step : 0), vy = mvy + (k ? c_nb[k - 1][1] * step : 0);
      int r[16];
      for (int i = 0; i < 16; i++) {
        const int x = 4 * bx + (i & 3), y = 4 * by + (i >> 2);
        r[i] = s.src[16 * y + x] - luma_at(s.win, x, y, vx, vy);
      }
      atomicAdd(&s.c9[k], satd4(r));
    }
    __syncthreads();
    int k = 0;
    for (int i = 1; i < 9; i++)
      if (s.c9[i] < s.c9[k]) k = i;
    if (k) { mvx += c_nb[k - 1][0] * step; mvy += c_nb[k - 1][1] * step; }
    if (step == 1 && t == 0) { s.mvx = mvx; s.mvy = mvy; s.icost = s.c9[k]; }
    __syncthreads();
  }
  for (int i = t; i < 384; i += 128) {
    if (i < 256) s.ipred[i] = luma_at(s.win, i & 15, i >> 4, mvx, mvy);
    else {
      const int p = (i - 256) / 64, j = (i - 256) % 64;
      s.ipred[i] = chroma_at(ref, l, p, 8 * mx + (j & 7), 8 * my + (j >> 3), mvx, mvy);
    }
  }
}

// Frame f's P picture flag and frame_num from the stream position.
__device__ __forceinline__ const int* frame_meta(const uint8_t* scratch, const Layout& l, int f) {
  return reinterpret_cast<const int*>(scratch + (int64_t)f * l.stride + l.meta);
}

// The macroblocks of wavefront line d: mbx + mby = d (slope 1) or mbx + 2 mby = d (slope 2); the k-th of them.
__device__ __forceinline__ bool line_mb(int d, int slope, int k, int wm, int hm, int& mx, int& my) {
  if (slope == 1) {
    if (d < 0 || d >= wm + hm - 1) return false;
    mx = max(0, d - hm + 1) + k;
    my = d - mx;
    return mx <= min(d, wm - 1);
  }
  if (d < 0 || d >= wm + 2 * hm - 2) return false;
  my = max(0, (d - wm + 2) / 2) + k;
  mx = d - 2 * my;
  return my <= min(d / 2, hm - 1);
}

// One launch per step of the wavefront over (frame, line): frame f runs line step - lag f (lag 0 when every frame is
// an IDR picture; LAG when a frame refers to the one before it, LAG_DB when it refers to the deblocked one).
//
// I4: the I_NxN candidate (Intra_4x4, 8.3.1) beside I_16x16.  Its 16 blocks run in decode order as a wavefront over
// bx + 2 by (10 steps, at most 2 blocks a step; a block's left, top, top-left and top-right lie on earlier steps):
// one thread per (block, mode) gives every available mode SATD(src - pred); one thread per block adds lambda * its
// mode bits (1 for predIntra4x4PredMode, else 4), takes the least cost (ties: the lower mode), and transforms,
// quantises (intra dead zone, all 16 coefficients) and reconstructs the block before the next step predicts from
// it.  Block 5 never takes modes 3 or 7, the only ones that read macroblock C (above right): C lies on the current
// macroblock's own anti-diagonal, so without them the wavefronts, lags and launches are those of the I_16x16 streams.
// I_NxN replaces I_16x16 when the sum of its block costs + I4_BIAS * lambda is below I_16x16's least luma SATD; in
// a P picture the cheaper intra candidate meets the inter one through INTRA_BIAS as I_16x16 alone did.  I_NxN falls
// back to I_PCM on MAX_LEVEL and PCM_BITS as I_16x16 does: its bits, like every coded macroblock's, never exceed
// PCM_BITS, so gab200_h264_bound / gab200_h264_p_bound and the slot strides hold for these streams as they are.
template <bool I4>
__global__ void __maxnreg__(80) h264_mb_kernel(int step, int lag, int slope, int f_lo, int qp, uint8_t* scratch,
                                                      const uint8_t* state, Layout l) {
  __shared__ std::conditional_t<I4, MbSharedI4, MbShared> s;
  const int f = f_lo + blockIdx.y, t = threadIdx.x;
  int mx, my;
  if (!line_mb(step - lag * f, slope, blockIdx.x, l.wm, l.hm, mx, my)) return;
  const int mb = my * l.wm + mx;
  const bool has_l = mx > 0, has_t = my > 0;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const Planes src(base + l.src, l), rec(base + l.rec, l);
  uint8_t* tot = base + l.tot;
  const int qpc = c_chroma_qp[qp];
  const bool is_p = frame_meta(scratch, l, f)[1] != 0;

  for (int i = t; i < 384; i += 128) {
    if (i < 256) s.src[i] = src.y[(16 * my + i / 16) * src.ys + 16 * mx + i % 16];
    else {
      const int p = (i - 256) / 64, j = (i - 256) % 64;
      s.src[i] = src.chroma(p)[(8 * my + j / 8) * src.cs + 8 * mx + j % 8];
    }
  }
  if (t < 32) {
    const int p = t < 16 ? 0 : 1 + (t - 16) / 8, j = t < 16 ? t : (t - 16) % 8;
    const uint8_t* pl = p == 0 ? rec.y : rec.chroma(p - 1);
    const int st = p == 0 ? rec.ys : rec.cs, n = p == 0 ? 16 : 8;
    s.top[t] = has_t ? pl[(n * my - 1) * st + n * mx + j] : 0;
    s.left[t] = has_l ? pl[(n * my + j) * st + n * mx - 1] : 0;
  }
  if (t >= 32 && t < 35) {
    const int p = t - 32;
    const uint8_t* pl = p == 0 ? rec.y : rec.chroma(p - 1);
    const int st = p == 0 ? rec.ys : rec.cs, n = p == 0 ? 16 : 8;
    s.tl[p] = has_t && has_l ? pl[(n * my - 1) * st + n * mx - 1] : 0;
  }
  if (t < 8) s.cost[t] = 0;
  if (t == 0) { s.maxlev = 0; s.bits = 0; s.inter = 0; }
  __syncthreads();
  if (is_p) {   // the reference: the previous frame of the batch (deblocked when the stream is), or the state's
    const Planes ref(f > 0 ? scratch + (int64_t)(f - 1) * l.stride + l.flt : const_cast<uint8_t*>(state) + 256, l);
    motion_search(s, ref, l, mx, my, qp);
  }

  // prediction parameters: DC values and the plane mode's a, b, c (8.3.3.3-4, 8.3.4.1-4)
  if (t == 0) {
    int st = 0, sl = 0, H = 0, V = 0;
    for (int i = 0; i < 16; i++) { st += s.top[i]; sl += s.left[i]; }
    s.par[0][0] = has_t && has_l ? (st + sl + 16) >> 5 : has_t ? (st + 8) >> 4 : has_l ? (sl + 8) >> 4 : 128;
    for (int x = 0; x < 8; x++) {
      H += (x + 1) * (s.top[8 + x] - (6 - x >= 0 ? s.top[6 - x] : s.tl[0]));
      V += (x + 1) * (s.left[8 + x] - (6 - x >= 0 ? s.left[6 - x] : s.tl[0]));
    }
    s.par[0][1] = 16 * (s.left[15] + s.top[15]);
    s.par[0][2] = (5 * H + 32) >> 6;
    s.par[0][3] = (5 * V + 32) >> 6;
  } else if (t == 32 || t == 64) {
    const int p = t / 32, o = 16 + 8 * (p - 1);
    const int* top = s.top + o;
    const int* left = s.left + o;
    for (int b = 0; b < 4; b++) {
      const int bx = b & 1, by = b >> 1;
      int st = 0, sl = 0;
      for (int i = 0; i < 4; i++) { st += top[4 * bx + i]; sl += left[4 * by + i]; }
      const int ts = (st + 2) >> 2, ls = (sl + 2) >> 2;
      int v;
      if (bx == by) v = has_t && has_l ? (st + sl + 4) >> 3 : has_t ? ts : has_l ? ls : 128;
      else if (bx == 1) v = has_t ? ts : has_l ? ls : 128;
      else v = has_l ? ls : has_t ? ts : 128;
      s.par[p][b] = v;
    }
    int H = 0, V = 0;
    for (int x = 0; x < 4; x++) {
      H += (x + 1) * (top[4 + x] - (2 - x >= 0 ? top[2 - x] : s.tl[p]));
      V += (x + 1) * (left[4 + x] - (2 - x >= 0 ? left[2 - x] : s.tl[p]));
    }
    s.par[p][4] = 16 * (left[7] + top[7]);
    s.par[p][5] = (34 * H + 32) >> 6;
    s.par[p][6] = (34 * V + 32) >> 6;
  }
  __syncthreads();

  // SATD of every mode: 64 luma (mode, block) tasks, 32 chroma (mode, plane, block) tasks
  if (t < 96) {
    int plane, mode, bx, by, so;
    if (t < 64) { plane = 0; mode = t / 16; bx = t & 3; by = (t >> 2) & 3; so = 0; }
    else { const int u = t - 64; mode = u / 8; plane = 1 + (u / 4) % 2; bx = u & 1; by = (u >> 1) & 1; so = 256 + 64 * (plane - 1); }
    const int n = plane == 0 ? 16 : 8;
    int r[16];
    for (int i = 0; i < 16; i++) {
      const int x = 4 * bx + (i & 3), y = 4 * by + (i >> 2);
      r[i] = s.src[so + y * n + x] - predict(s, plane, mode, x, y);
    }
    atomicAdd(&s.cost[plane == 0 ? mode : 4 + mode], satd4(r));
  }
  if constexpr (I4) {
    if (t == 0) { s.own = 0; s.sum4 = 0; s.mbits4 = 0; s.max4 = 0; }
    const int* info = reinterpret_cast<const int*>(base + l.info);
    const uint64_t* modes = reinterpret_cast<const uint64_t*>(base + l.modes);
    const int L = lambda_of(qp);
    // the 4x4 block's edge (see pred4) and which of its samples exist, in the order left, top, top-right
    auto edge = [&](int bx, int by, int* e, bool& al, bool& at) {
      al = bx > 0 || has_l;
      at = by > 0 || has_t;
      const bool atr = bx < 3 && (by == 0 ? has_t : blk_idx(bx + 1, by - 1) < blk_idx(bx, by));
      const int x0 = 4 * bx, y0 = 4 * by;
      auto p = [&](int x, int y) {   // the reconstructed sample at (x, y) of the macroblock, x, y >= -1
        return y < 0 ? (x < 0 ? s.tl[0] : s.top[x]) : x < 0 ? s.left[y] : s.r4[16 * y + x];
      };
      for (int j = 0; j < 4; j++) e[3 - j] = al ? p(x0 - 1, y0 + j) : 0;
      e[4] = al && at ? p(x0 - 1, y0 - 1) : 0;
      for (int i = 0; i < 8; i++) e[5 + i] = at ? p(i < 4 || atr ? x0 + i : x0 + 3, y0 - 1) : 0;
    };
    auto dc4 = [](const int* e, bool al, bool at) {
      const int sl = e[0] + e[1] + e[2] + e[3], st = e[5] + e[6] + e[7] + e[8];
      return al && at ? (sl + st + 4) >> 3 : at ? (st + 2) >> 2 : al ? (sl + 2) >> 2 : 128;
    };
    for (int st = 0; st < 10; st++) {
      const int by_lo = max(0, (st - 2) / 2);   // blocks (st - 2 by, by) with 0 <= st - 2 by <= 3
      __syncthreads();
      if (t < 18) {
        const int by = by_lo + t / 9, bx = st - 2 * by, m = t % 9;
        if (by <= 3 && bx >= 0) {
          int e[13];
          bool al, at;
          edge(bx, by, e, al, at);
          // 8.3.1.2's availability; block 5 never takes modes 3 and 7 (macroblock C)
          const bool ok = m == 2 || (m == 1 || m == 8 ? al
                                     : m == 0 ? at
                                     : m == 3 || m == 7 ? at && !(bx == 3 && by == 0)
                                     : al && at);
          int cost = INT_MAX;
          if (ok) {
            const int dc = dc4(e, al, at);
            int r[16];
            for (int i = 0; i < 16; i++)
              r[i] = s.src[16 * (4 * by + (i >> 2)) + 4 * bx + (i & 3)] - pred4(e, m, dc, i & 3, i >> 2);
            cost = satd4(r);
          }
          s.c4[t / 9][m] = cost;
        }
      }
      __syncthreads();
      if (t < 2) {
        const int by = by_lo + t, bx = st - 2 * by;
        if (by <= 3 && bx >= 0) {
          const int pm = i4_pred_mode(s.own, info, modes, l.wm, mx, my, bx, by);
          int m = 0, best = INT_MAX;
          for (int k = 0; k < 9; k++) {
            if (s.c4[t][k] == INT_MAX) continue;
            const int c = s.c4[t][k] + L * (k == pm ? 1 : 4);
            if (c < best) { best = c; m = k; }
          }
          int e[13];
          bool al, at;
          edge(bx, by, e, al, at);
          const int dc = dc4(e, al, at), b = 4 * by + bx;
          int pr[16], x[16], w[16];
          for (int i = 0; i < 16; i++) {
            pr[i] = pred4(e, m, dc, i & 3, i >> 2);
            x[i] = s.src[16 * (4 * by + (i >> 2)) + 4 * bx + (i & 3)] - pr[i];
          }
          for (int i = 0; i < 4; i++)      // CF x CF^T
            for (int j = 0; j < 4; j++) {
              const int a = x[j], b1 = x[4 + j], c = x[8 + j], d = x[12 + j];
              w[i * 4 + j] = i == 0 ? a + b1 + c + d : i == 1 ? 2 * a + b1 - c - 2 * d
                             : i == 2 ? a - b1 - c + d : a - 2 * b1 + 2 * c - d;
            }
          const int qbits = 15 + qp / 6, fq = (1 << qbits) / 3;
          int nz = 0, mx_ = 0, dq[16];
          for (int i = 0; i < 4; i++) {
            const int a = w[4 * i], b1 = w[4 * i + 1], c = w[4 * i + 2], d = w[4 * i + 3];
            const int w4[4] = {a + b1 + c + d, 2 * a + b1 - c - 2 * d, a - b1 - c + d, a - 2 * b1 + 2 * c - d};
            for (int j = 0; j < 4; j++) {
              const int k = 4 * i + j, lv = quant(w4[j], c_mf[qp % 6][pos_class(k)], qbits, fq);
              const int ls = 16 * c_v[qp % 6][pos_class(k)];
              s.lev[b][k] = lv;
              nz += lv != 0;
              mx_ = max(mx_, abs(lv));
              dq[k] = qp >= 24 ? (lv * ls) << (qp / 6 - 4) : (lv * ls + (1 << (3 - qp / 6))) >> (4 - qp / 6);
            }
          }
          idct4(dq);
          for (int i = 0; i < 16; i++) s.r4[16 * (4 * by + (i >> 2)) + 4 * bx + (i & 3)] = clip255(pr[i] + dq[i]);
          s.tot[b] = nz;
          atomicMax(&s.max4, mx_);
          atomicAdd(&s.sum4, best);
          atomicAdd(&s.mbits4, m == pm ? 1 : 4);
          atomicOr(reinterpret_cast<unsigned long long*>(&s.own), (unsigned long long)m << (4 * b));
        }
      }
    }
  }
  __syncthreads();
  if (t == 0) {
    const bool lav[4] = {has_t, has_l, true, has_t && has_l};
    const bool cav[4] = {true, has_l, has_t, has_t && has_l};
    int lm = 2, cm = 0;
    for (int m = 0; m < 4; m++) {
      if (lav[m] && (s.cost[m] < s.cost[lm] || (s.cost[m] == s.cost[lm] && m < lm))) lm = m;
      if (cav[m] && (s.cost[4 + m] < s.cost[4 + cm] || (s.cost[4 + m] == s.cost[4 + cm] && m < cm))) cm = m;
    }
    s.lmode = lm;
    s.cmode = cm;
    int intra = s.cost[lm];
    if constexpr (I4) {
      s.nxn = s.sum4 + I4_BIAS * lambda_of(qp) < intra;
      if (s.nxn) intra = s.sum4 + I4_BIAS * lambda_of(qp);
    }
    s.inter = is_p && !(intra + INTRA_BIAS * lambda_of(qp) < s.icost);
    if constexpr (I4) {
      s.nxn = s.nxn && !s.inter;
      if (s.nxn) s.maxlev = s.max4;
    }
  }
  __syncthreads();
  const bool inter = s.inter;
  bool nxn = false;
  if constexpr (I4) nxn = s.nxn;
  for (int i = t; i < 384; i += 128) {
    if (inter) s.pred[i] = s.ipred[i];
    else if (i < 256) s.pred[i] = predict(s, 0, s.lmode, i & 15, i >> 4);
    else { const int p = 1 + (i - 256) / 64, j = (i - 256) % 64; s.pred[i] = predict(s, p, s.cmode, j & 7, j >> 3); }
  }
  __syncthreads();

  // forward transform and quantisation: one thread per 4x4 block (16 luma raster, 4 Cb, 4 Cr); the dead zone is
  // f = 2^qbits / 3 for intra, 2^qbits / 6 for inter; an inter luma block keeps its DC coefficient (an I_NxN
  // macroblock's luma blocks are already coded)
  if (t < 24 && !(nxn && t < 16)) {
    const bool luma = t < 16;
    const int bx = luma ? (t & 3) : (t & 1), by = luma ? (t >> 2) : ((t >> 1) & 1);
    const int n = luma ? 16 : 8, so = luma ? 0 : 256 + 64 * ((t - 16) / 4);
    const int q = luma ? qp : qpc;
    int x[16], m[16];
    for (int i = 0; i < 16; i++) {
      const int o = so + (4 * by + (i >> 2)) * n + 4 * bx + (i & 3);
      x[i] = s.src[o] - s.pred[o];
    }
    for (int i = 0; i < 4; i++)      // m = CF x (columns)
      for (int j = 0; j < 4; j++) {
        const int a = x[j], b = x[4 + j], c = x[8 + j], e = x[12 + j];
        m[i * 4 + j] = i == 0 ? a + b + c + e : i == 1 ? 2 * a + b - c - 2 * e : i == 2 ? a - b - c + e : a - 2 * b + 2 * c - e;
      }
    const int qbits = 15 + q / 6, fq = (1 << qbits) / (inter ? 6 : 3);
    const int k0 = inter && luma ? 0 : 1;
    int nz = 0, mx_ = 0;
    for (int i = 0; i < 4; i++) {    // w = m CF^T (rows)
      const int a = m[4 * i], b = m[4 * i + 1], c = m[4 * i + 2], e = m[4 * i + 3];
      const int w4[4] = {a + b + c + e, 2 * a + b - c - 2 * e, a - b - c + e, a - 2 * b + 2 * c - e};
      for (int j = 0; j < 4; j++) {
        const int k = 4 * i + j;
        s.w[t][k] = w4[j];
        const int lv = k < k0 ? 0 : quant(w4[j], c_mf[q % 6][pos_class(k)], qbits, fq);
        s.lev[t][k] = lv;
        nz += lv != 0;
        mx_ = max(mx_, abs(lv));
      }
    }
    s.tot[t] = nz;
    atomicMax(&s.maxlev, mx_);
  }
  __syncthreads();

  // DC transforms, quantisation and their dequantisation (8.5.10, 8.5.11)
  if (t == 0 && !inter && !nxn) {
    int a[16], b[16];
    for (int i = 0; i < 16; i++) a[i] = s.w[i][0];   // [by * 4 + bx]
    // b = HD a HD, >> 1
    for (int j = 0; j < 4; j++) {
      const int p0 = a[j], p1 = a[4 + j], p2 = a[8 + j], p3 = a[12 + j];
      b[j] = p0 + p1 + p2 + p3; b[4 + j] = p0 + p1 - p2 - p3; b[8 + j] = p0 - p1 - p2 + p3; b[12 + j] = p0 - p1 + p2 - p3;
    }
    const int qbits = 15 + qp / 6, fq = (1 << qbits) / 3;
    int mx_ = 0;
    for (int i = 0; i < 4; i++) {
      const int p0 = b[4 * i], p1 = b[4 * i + 1], p2 = b[4 * i + 2], p3 = b[4 * i + 3];
      const int r4[4] = {p0 + p1 + p2 + p3, p0 + p1 - p2 - p3, p0 - p1 - p2 + p3, p0 - p1 + p2 - p3};
      for (int j = 0; j < 4; j++) {
        const int lv = quant(r4[j] >> 1, c_mf[qp % 6][0], qbits + 1, 2 * fq);
        s.dc[4 * i + j] = lv;
        mx_ = max(mx_, abs(lv));
      }
    }
    atomicMax(&s.maxlev, mx_);
    // inverse: f = HD c HD, then scaled
    for (int j = 0; j < 4; j++) {
      const int p0 = s.dc[j], p1 = s.dc[4 + j], p2 = s.dc[8 + j], p3 = s.dc[12 + j];
      b[j] = p0 + p1 + p2 + p3; b[4 + j] = p0 + p1 - p2 - p3; b[8 + j] = p0 - p1 - p2 + p3; b[12 + j] = p0 - p1 + p2 - p3;
    }
    const int ls = 16 * c_v[qp % 6][0];
    for (int i = 0; i < 4; i++) {
      const int p0 = b[4 * i], p1 = b[4 * i + 1], p2 = b[4 * i + 2], p3 = b[4 * i + 3];
      const int r4[4] = {p0 + p1 + p2 + p3, p0 + p1 - p2 - p3, p0 - p1 - p2 + p3, p0 - p1 + p2 - p3};
      for (int j = 0; j < 4; j++)
        s.dcr[4 * i + j] = qp >= 36 ? (r4[j] * ls) << (qp / 6 - 6) : (r4[j] * ls + (1 << (5 - qp / 6))) >> (6 - qp / 6);
    }
  } else if (t == 32 || t == 64) {
    const int p = t / 64, o = 16 + 4 * p;
    const int a0 = s.w[o][0], a1 = s.w[o + 1][0], a2 = s.w[o + 2][0], a3 = s.w[o + 3][0];
    const int c4[4] = {a0 + a1 + a2 + a3, a0 - a1 + a2 - a3, a0 + a1 - a2 - a3, a0 - a1 - a2 + a3};
    const int qbits = 15 + qpc / 6, fq = (1 << qbits) / (inter ? 6 : 3);
    int mx_ = 0;
    for (int i = 0; i < 4; i++) {
      s.cdc[p][i] = quant(c4[i], c_mf[qpc % 6][0], qbits + 1, 2 * fq);
      mx_ = max(mx_, abs(s.cdc[p][i]));
    }
    atomicMax(&s.maxlev, mx_);
    const int l0 = s.cdc[p][0], l1 = s.cdc[p][1], l2 = s.cdc[p][2], l3 = s.cdc[p][3];
    const int f4[4] = {l0 + l1 + l2 + l3, l0 - l1 + l2 - l3, l0 + l1 - l2 - l3, l0 - l1 - l2 + l3};
    const int ls = 16 * c_v[qpc % 6][0];
    for (int i = 0; i < 4; i++) s.cdcr[p][i] = ((f4[i] * ls) << (qpc / 6)) >> 5;
  }
  __syncthreads();

  // reconstruction: dequantise, inverse transform, add the prediction
  if (t < 24 && !(nxn && t < 16)) {
    const bool luma = t < 16;
    const int q = luma ? qp : qpc;
    int dq[16];
    for (int k = 0; k < 16; k++) {
      const int ls = 16 * c_v[q % 6][pos_class(k)], c = s.lev[t][k];
      dq[k] = q >= 24 ? (c * ls) << (q / 6 - 4) : (c * ls + (1 << (3 - q / 6))) >> (4 - q / 6);
    }
    if (!(inter && luma)) dq[0] = luma ? s.dcr[t] : s.cdcr[(t - 16) / 4][(t - 16) & 3];
    idct4(dq);
    for (int k = 0; k < 16; k++) s.w[t][k] = dq[k];   // the residual
  }
  __syncthreads();
  if (t == 0) {
    int al = 0, ac = 0, dcc = 0, m8 = 0;
    for (int i = 0; i < 16; i++) {
      al += s.tot[i];
      if (s.tot[i]) m8 |= 1 << (((i >> 3) << 1) | ((i & 3) >> 1));   // the block's 8x8 quadrant
    }
    for (int i = 16; i < 24; i++) ac += s.tot[i];
    for (int i = 0; i < 8; i++) dcc |= s.cdc[i / 4][i % 4];
    s.cbpl = inter || nxn ? m8 : al ? 15 : 0;
    s.cbpc = ac ? 2 : dcc ? 1 : 0;
  }
  __syncthreads();
  // TotalCoeff of this macroblock's blocks (nC of its own later blocks reads them): luma by luma4x4 raster position
  if (t < 24) tot[(int64_t)mb * 24 + t] = (uint8_t)s.tot[t];
  __syncthreads();

  // CAVLC bit count, one thread per residual block: 0 luma DC, 1..16 luma AC (luma4x4BlkIdx order; an inter block's
  // 16 coefficients), 17/18 Cb/Cr DC, 19..26 Cb AC, 23..26 Cr AC; the levels in scan order go to the writer
  const int info = s.lmode | s.cmode << 2 | s.cbpc << 4 | (!inter && !nxn && s.cbpl ? 1 : 0) << 6 | inter << 8 |
                   (inter || nxn ? s.cbpl : 0) << 9 | nxn << 14;
  if (t < BLOCKS) {
    int c[16], plane, x, y, maxn;
    block_geom(t, mx, my, plane, x, y, maxn);
    if (t == 0) for (int k = 0; k < 16; k++) c[k] = s.dc[c_zigzag[k]];
    else if (t <= 16) {
      const int b = c_blk_y[t - 1] * 4 + c_blk_x[t - 1];
      if (inter || nxn) maxn = 16;
      for (int k = 0; k < maxn; k++) c[k] = s.lev[b][c_zigzag[k + 16 - maxn]];
    }
    else if (t <= 18) for (int k = 0; k < 4; k++) c[k] = s.cdc[t - 17][k];
    else { const int b = 16 + (t - 19); for (int k = 0; k < 15; k++) c[k] = s.lev[b][c_zigzag[k + 1]]; }
    int16_t* out = reinterpret_cast<int16_t*>(base + l.lev) + ((int64_t)mb * BLOCKS + t) * 16;
    for (int k = 0; k < maxn; k++) out[k] = (int16_t)max(-32768, min(32767, c[k]));
    if (s.maxlev <= MAX_LEVEL && block_present(t, info)) {
      BitSink sink{nullptr, 0, 0};
      const int nc = plane < 0 ? -1 : nc_of(tot, l, plane, x, y);
      atomicAdd(&s.bits, cavlc_block(c, maxn, nc, sink));
    }
  }
  __syncthreads();
  if (t == 0) {
    int hb = mb_header_bits(info, is_p);
    if constexpr (I4) {
      reinterpret_cast<uint64_t*>(base + l.modes)[mb] = s.own;
      const int cbp = s.cbpl | s.cbpc << 4;
      if (nxn) hb = (is_p ? 5 : 1) + s.mbits4 + ue_bits(s.cmode) + ue_bits(c_intra_cbp[cbp]) + (cbp ? 1 : 0);
    }
    const int bits = s.bits + hb;
    s.pcm = s.maxlev > MAX_LEVEL || bits > PCM_BITS;
    reinterpret_cast<int*>(base + l.info)[mb] = s.pcm ? (1 << 7) : info;
    reinterpret_cast<int*>(base + l.bits)[mb] = s.pcm ? 0 : bits;
    reinterpret_cast<int*>(base + l.mv)[mb] = inter && !s.pcm ? (s.mvx & 0xffff) | (int)((unsigned)s.mvy << 16) : 0;
  }
  __syncthreads();
  if (s.pcm && t < 24) tot[(int64_t)mb * 24 + t] = 16;
  for (int i = t; i < 384; i += 128) {
    int v;
    if (s.pcm) v = s.src[i];
    else if (nxn && i < 256) {
      if constexpr (I4) v = s.r4[i];
    } else if (i < 256) v = clip255(s.pred[i] + s.w[((i >> 4) >> 2) * 4 + ((i & 15) >> 2)][((i >> 4) & 3) * 4 + (i & 3)]);
    else {
      const int p = (i - 256) / 64, j = (i - 256) % 64, x = j & 7, y = j >> 3;
      v = clip255(s.pred[i] + s.w[16 + 4 * p + (y >> 2) * 2 + (x >> 2)][(y & 3) * 4 + (x & 3)]);
    }
    if (i < 256) rec.y[(16 * my + (i >> 4)) * rec.ys + 16 * mx + (i & 15)] = (uint8_t)v;
    else {
      const int p = (i - 256) / 64, j = (i - 256) % 64;
      rec.chroma(p)[(8 * my + (j >> 3)) * rec.cs + 8 * mx + (j & 7)] = (uint8_t)v;
    }
  }
}

// ---- the deblocking filter (8.7) ---------------------------------------------------------------------------------
// Tables 8-16 (alpha', beta') and 8-17 (tC0 at bS 1, 2, 3), indexed by indexA = indexB = qPav (offsets 0).
__constant__ uint8_t c_alpha[52] = {0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,   0,   0,   0,   0,   0,   4,   4,
                                    5,  6,  7,  8,  9,  10, 12, 13, 15, 17, 20,  22,  25,  28,  32,  36,  40,  45,
                                    50, 56, 63, 71, 80, 90, 101, 113, 127, 144, 162, 182, 203, 226, 255, 255};
__constant__ uint8_t c_beta[52] = {0, 0, 0, 0, 0, 0, 0, 0, 0,  0,  0,  0,  0,  0,  0,  0,  2,  2,  2,  3,  3,  3,  3,  4,  4,  4,
                                   6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17, 17, 18, 18};
__constant__ uint8_t c_tc0[52][3] = {
    {0, 0, 0}, {0, 0, 0}, {0, 0, 0},   {0, 0, 0},   {0, 0, 0},    {0, 0, 0},    {0, 0, 0},    {0, 0, 0},
    {0, 0, 0}, {0, 0, 0}, {0, 0, 0},   {0, 0, 0},   {0, 0, 0},    {0, 0, 0},    {0, 0, 0},    {0, 0, 0},
    {0, 0, 0}, {0, 0, 1}, {0, 0, 1},   {0, 0, 1},   {0, 0, 1},    {0, 1, 1},    {0, 1, 1},    {1, 1, 1},
    {1, 1, 1}, {1, 1, 1}, {1, 1, 1},   {1, 1, 2},   {1, 1, 2},    {1, 1, 2},    {1, 1, 2},    {1, 2, 3},
    {1, 2, 3}, {2, 2, 3}, {2, 2, 4},   {2, 3, 4},   {2, 3, 4},    {3, 3, 5},    {3, 4, 6},    {3, 4, 6},
    {4, 5, 7}, {4, 5, 8}, {4, 6, 9},   {5, 7, 10},  {6, 8, 11},   {6, 8, 13},   {7, 10, 14},  {8, 11, 16},
    {9, 12, 18}, {10, 13, 20}, {11, 15, 23}, {13, 17, 25}};

// One line of samples across an edge: q points at q0, p_i = q[-(i + 1) step], q_i = q[i step] (8.7.2.3, 8.7.2.4).
__device__ __forceinline__ void filter_line(uint8_t* q, int step, bool chroma, int bS, int qpav) {
  const int alpha = c_alpha[qpav], beta = c_beta[qpav];
  const int p0 = q[-step], p1 = q[-2 * step], q0 = q[0], q1 = q[step];
  if (!(abs(p0 - q0) < alpha && abs(p1 - p0) < beta && abs(q1 - q0) < beta)) return;
  if (chroma) {
    if (bS < 4) {
      const int tc = c_tc0[qpav][bS - 1] + 1;
      const int delta = min(max((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc), tc);
      q[-step] = (uint8_t)clip255(p0 + delta);
      q[0] = (uint8_t)clip255(q0 - delta);
    } else {
      q[-step] = (uint8_t)((2 * p1 + p0 + q1 + 2) >> 2);
      q[0] = (uint8_t)((2 * q1 + q0 + p1 + 2) >> 2);
    }
    return;
  }
  const int p2 = q[-3 * step], q2 = q[2 * step];
  const bool ap = abs(p2 - p0) < beta, aq = abs(q2 - q0) < beta;
  if (bS < 4) {
    const int tc0 = c_tc0[qpav][bS - 1], tc = tc0 + ap + aq;
    const int delta = min(max((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc), tc);
    q[-step] = (uint8_t)clip255(p0 + delta);
    q[0] = (uint8_t)clip255(q0 - delta);
    if (ap) q[-2 * step] = (uint8_t)(p1 + min(max((p2 + ((p0 + q0 + 1) >> 1) - (p1 << 1)) >> 1, -tc0), tc0));
    if (aq) q[step] = (uint8_t)(q1 + min(max((q2 + ((p0 + q0 + 1) >> 1) - (q1 << 1)) >> 1, -tc0), tc0));
    return;
  }
  const bool strong = abs(p0 - q0) < ((alpha >> 2) + 2);
  if (ap && strong) {
    const int p3 = q[-4 * step];
    q[-step] = (uint8_t)((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
    q[-2 * step] = (uint8_t)((p2 + p1 + p0 + q0 + 2) >> 2);
    q[-3 * step] = (uint8_t)((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
  } else {
    q[-step] = (uint8_t)((2 * p1 + p0 + q1 + 2) >> 2);
  }
  if (aq && strong) {
    const int q3 = q[3 * step];
    q[0] = (uint8_t)((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
    q[step] = (uint8_t)((p0 + q0 + q1 + q2 + 2) >> 2);
    q[2 * step] = (uint8_t)((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3);
  } else {
    q[0] = (uint8_t)((2 * q1 + q0 + p1 + 2) >> 2);
  }
}

// One warp per macroblock (x, y) on line x + 2 y = step - lag f - DB_LAG of frame f: the macroblock's samples from
// rec (no filtering has reached them yet), the 4 columns left of it and the 4 rows above it from flt (their
// macroblocks' filtering is done); bS of every 4-sample edge segment, then the vertical edges left to right (one lane
// per row: 16 luma, 8 Cb, 8 Cr), then the horizontal edges top to bottom (one lane per column); the samples the
// filter may have changed go back to flt.
__global__ void __launch_bounds__(32) h264_deblock_kernel(int step, int lag, int f_lo, int qp, uint8_t* scratch,
                                                          Layout l) {
  __shared__ uint8_t sy[20][20];        // luma rows and columns -4 .. 15
  __shared__ uint8_t sc[2][10][10];     // chroma rows and columns -2 .. 7
  __shared__ uint8_t sbs[2][4][4];      // [vertical, horizontal][edge][segment]
  const int f = f_lo + blockIdx.y, t = threadIdx.x;
  int mx, my;
  if (!line_mb(step - lag * f - DB_LAG, 2, blockIdx.x, l.wm, l.hm, mx, my)) return;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const uint8_t* rec = base + l.rec;
  uint8_t* flt = base + l.flt;
  const int ys = 16 * l.wm, cs = 8 * l.wm;
  const int64_t c0 = (int64_t)ys * 16 * l.hm, cpl = (int64_t)cs * 8 * l.hm;   // Cb's offset, a chroma plane's bytes
  const bool has_l = mx > 0, has_t = my > 0;
  for (int i = t; i < 400; i += 32) {
    const int r = i / 20 - 4, c = i % 20 - 4;
    if ((r < 0 && (c < 0 || !has_t)) || (c < 0 && !has_l)) continue;
    sy[r + 4][c + 4] = (r < 0 || c < 0 ? flt : rec)[(int64_t)(16 * my + r) * ys + 16 * mx + c];
  }
  for (int i = t; i < 200; i += 32) {
    const int p = i / 100, r = i % 100 / 10 - 2, c = i % 10 - 2;
    if ((r < 0 && (c < 0 || !has_t)) || (c < 0 && !has_l)) continue;
    sc[p][r + 2][c + 2] = (r < 0 || c < 0 ? flt : rec)[c0 + p * cpl + (int64_t)(8 * my + r) * cs + 8 * mx + c];
  }
  // bS (8.7.2.1): one lane per (direction, edge, segment)
  const int* info = reinterpret_cast<const int*>(base + l.info);
  const int* mv = reinterpret_cast<const int*>(base + l.mv);
  const uint8_t* tot = base + l.tot;
  const int mb = my * l.wm + mx, mb_l = mb - 1, mb_t = mb - l.wm;
  {
    const int dir = t >> 4, e = (t >> 2) & 3, seg = t & 3;
    const int qbx = dir ? seg : e, qby = dir ? e : seg;
    const int nb = e ? mb : dir ? mb_t : mb_l;
    const int pbx = dir ? seg : (e ? e - 1 : 3), pby = dir ? (e ? e - 1 : 3) : seg;
    int bS = 0;
    if (e || (dir ? has_t : has_l)) {
      const bool intra = !((info[mb] >> 8) & 1) || !((info[nb] >> 8) & 1);
      if (intra) bS = e ? 3 : 4;
      else if (tot[(int64_t)mb * 24 + qby * 4 + qbx] || tot[(int64_t)nb * 24 + pby * 4 + pbx]) bS = 2;
      else {
        const int a = mv[mb], b = mv[nb];
        bS = abs((int16_t)(a & 0xffff) - (int16_t)(b & 0xffff)) >= 4 || abs((a >> 16) - (b >> 16)) >= 4;
      }
    }
    sbs[dir][e][seg] = (uint8_t)bS;
  }
  // qP: the stream QP, 0 on an I_PCM side; chroma averages each side's QPc
  const int qp_q = (info[mb] >> 7) & 1 ? 0 : qp;
  const int qp_l = has_l && !((info[mb_l] >> 7) & 1) ? qp : 0, qp_t = has_t && !((info[mb_t] >> 7) & 1) ? qp : 0;
  __syncwarp();
  for (int dir = 0; dir < 2; dir++) {
    const int qp_p = dir ? qp_t : qp_l;
    if (t < 16) {
      for (int e = 0; e < 4; e++) {
        const int bS = sbs[dir][e][t >> 2];
        if (bS) filter_line(dir ? &sy[4 * e + 4][t + 4] : &sy[t + 4][4 * e + 4], dir ? 20 : 1, false, bS,
                            e ? qp_q : (qp_p + qp_q + 1) >> 1);
      }
    } else {
      const int p = (t - 16) >> 3, k = t & 7;
      for (int e = 0; e < 2; e++) {
        const int bS = sbs[dir][2 * e][k >> 1];
        const int qc = c_chroma_qp[qp_q];
        if (bS) filter_line(dir ? &sc[p][4 * e + 2][k + 2] : &sc[p][k + 2][4 * e + 2], dir ? 10 : 1, true, bS,
                            e ? qc : (c_chroma_qp[qp_p] + qc + 1) >> 1);
      }
    }
    __syncwarp();
  }
  for (int i = t; i < 361; i += 32) {   // rows and columns -3 .. 15, the corner excepted
    const int r = i / 19 - 3, c = i % 19 - 3;
    if ((r < 0 && (c < 0 || !has_t)) || (c < 0 && !has_l)) continue;
    flt[(int64_t)(16 * my + r) * ys + 16 * mx + c] = sy[r + 4][c + 4];
  }
  for (int i = t; i < 162; i += 32) {   // rows and columns -1 .. 7
    const int p = i / 81, r = i % 81 / 9 - 1, c = i % 9 - 1;
    if ((r < 0 && (c < 0 || !has_t)) || (c < 0 && !has_l)) continue;
    flt[c0 + p * cpl + (int64_t)(8 * my + r) * cs + 8 * mx + c] = sc[p][r + 2][c + 2];
  }
}

// ---- P slices: vector prediction and skip runs, after every decision is made -------------------------------------
struct Neighbour {
  bool avail;
  int ref, x, y;   // ref 0 for an inter macroblock, -1 for an intra one or none
};

__device__ Neighbour neighbour(const int* info, const int* mv, const Layout& l, int x, int y) {
  if (x < 0 || y < 0 || x >= l.wm) return {false, -1, 0, 0};
  const int mb = y * l.wm + x;
  if (!((info[mb] >> 8) & 1)) return {true, -1, 0, 0};
  const int v = mv[mb];
  return {true, 0, (int)(int16_t)(v & 0xffff), v >> 16};
}

__device__ __forceinline__ int median3(int a, int b, int c) { return max(min(a, b), min(max(a, b), c)); }

// 8.4.1.3 (mvp of a 16x16 partition with refIdx 0) and 8.4.1.1 (P_Skip); one thread per macroblock.  A P_L0_16x16
// macroblock with no coded coefficient whose vector equals its mvpSkip becomes P_Skip; the others get their mvd bits.
__global__ void __launch_bounds__(128) h264_mvp_kernel(uint8_t* scratch, Layout l) {
  const int f = blockIdx.y, mb = blockIdx.x * blockDim.x + threadIdx.x;
  if (mb >= l.nmb || !frame_meta(scratch, l, f)[1]) return;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  int* info = reinterpret_cast<int*>(base + l.info);
  const int* mv = reinterpret_cast<const int*>(base + l.mv);
  const int me = info[mb];
  if (!((me >> 8) & 1)) return;
  const int x = mb % l.wm, y = mb / l.wm;
  const Neighbour A = neighbour(info, mv, l, x - 1, y);
  Neighbour B = neighbour(info, mv, l, x, y - 1);
  Neighbour C = neighbour(info, mv, l, x + 1, y - 1);
  if (!C.avail) C = neighbour(info, mv, l, x - 1, y - 1);
  const bool skip0 = !A.avail || !B.avail || (A.ref == 0 && A.x == 0 && A.y == 0) || (B.ref == 0 && B.x == 0 && B.y == 0);
  if (!B.avail && !C.avail && A.avail) B = C = A;
  int px, py;
  const int n = (A.ref == 0) + (B.ref == 0) + (C.ref == 0);
  if (n == 1) {
    const Neighbour& o = A.ref == 0 ? A : B.ref == 0 ? B : C;
    px = o.x; py = o.y;
  } else {
    px = median3(A.x, B.x, C.x);
    py = median3(A.y, B.y, C.y);
  }
  const int vx = (int)(int16_t)(mv[mb] & 0xffff), vy = mv[mb] >> 16;
  const int sx = skip0 ? 0 : px, sy = skip0 ? 0 : py;
  int* bits = reinterpret_cast<int*>(base + l.bits);
  if (inter_cbp(me) == 0 && vx == sx && vy == sy) {
    info[mb] = me | 1 << 13;
    bits[mb] = 0;
    return;
  }
  const int dx = vx - px, dy = vy - py;
  reinterpret_cast<int*>(base + l.mvd)[mb] = (dx & 0xffff) | (int)((unsigned)dy << 16);
  bits[mb] += se_bits(dx) + se_bits(dy);
}

// Each coded macroblock's mb_skip_run (the P_Skip macroblocks just before it) and the slice's trailing run, which the
// last macroblock carries when it is skipped; one thread per macroblock.
__global__ void __launch_bounds__(128) h264_run_kernel(uint8_t* scratch, Layout l) {
  const int f = blockIdx.y, mb = blockIdx.x * blockDim.x + threadIdx.x;
  if (mb >= l.nmb || !frame_meta(scratch, l, f)[1]) return;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const int* info = reinterpret_cast<const int*>(base + l.info);
  const bool skipped = (info[mb] >> 13) & 1;
  if (skipped && mb != l.nmb - 1) return;
  int r = 0;
  while (r < mb && ((info[mb - 1 - r] >> 13) & 1)) r++;
  if (skipped) r++;
  reinterpret_cast<int*>(base + l.run)[mb] = r;
  if (!((info[mb] >> 7) & 1)) reinterpret_cast<int*>(base + l.bits)[mb] += ue_bits(r);
}

// ---- bit offsets -------------------------------------------------------------------------------------------------
// x -> x + a (ceil == 0) or ceil8(x + a) + b (ceil == 1)
struct Map {
  int a, b, ceil;
};

__device__ __forceinline__ Map compose(Map f, Map g) {   // g after f
  if (!g.ceil) return f.ceil ? Map{f.a, f.b + g.a, 1} : Map{f.a + g.a, 0, 0};
  if (!f.ceil) return Map{f.a + g.a, g.b, 1};
  return Map{f.a, ((f.b + g.a + 7) & ~7) + g.b, 1};
}

__device__ __forceinline__ int apply(Map m, int x) { return m.ceil ? ((x + m.a + 7) & ~7) + m.b : x + m.a; }

__global__ void __launch_bounds__(1024) h264_scan_kernel(uint8_t* scratch, Layout l) {
  __shared__ Map part[1024];
  __shared__ int s_total;
  const int f = blockIdx.x, t = threadIdx.x;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const int* info = reinterpret_cast<const int*>(base + l.info);
  const int* bits = reinterpret_cast<const int*>(base + l.bits);
  const int* run = reinterpret_cast<const int*>(base + l.run);
  int* off = reinterpret_cast<int*>(base + l.off);
  const int* meta = frame_meta(scratch, l, f);
  const bool is_p = meta[1] != 0;
  const int header = is_p ? P_HEADER_BITS : HEADER_BITS;
  // an I_PCM macroblock: its skip run, ue(mb_type), then its samples byte-aligned
  auto map = [&](int i) {
    return (info[i] >> 7) & 1 ? Map{(is_p ? ue_bits(run[i]) : 0) + 9, PCM_BITS - 9, 1} : Map{bits[i], 0, 0};
  };
  const int per = (l.nmb + 1023) / 1024, lo = min(t * per, l.nmb), hi = min(lo + per, l.nmb);
  Map m{0, 0, 0};
  for (int i = lo; i < hi; i++) m = compose(m, map(i));
  part[t] = m;
  __syncthreads();
  for (int s = 1; s < 1024; s <<= 1) {   // inclusive Hillis-Steele scan
    const Map prev = t >= s ? part[t - s] : Map{0, 0, 0};
    __syncthreads();
    if (t >= s) part[t] = compose(prev, part[t]);
    __syncthreads();
  }
  int x = t == 0 ? header : apply(part[t - 1], header);
  for (int i = lo; i < hi; i++) {
    off[i] = x;
    x = apply(map(i), x);
  }
  if (t == 1023) s_total = apply(part[1023], header);
  __syncthreads();
  const int total = s_total;                       // bits before the stop bit
  const int nbytes = (total + 1 + 7) / 8;
  uint32_t* raw = reinterpret_cast<uint32_t*>(base + l.raw);
  for (int i = t; i < (nbytes + 3) / 4 + 1; i += 1024) raw[i] = 0;
  __syncthreads();
  if (t == 0) {
    // first_mb_in_slice 0, slice_type 7, pps 0, frame_num 0000, idr_pic_id 1, two flags, slice_qp_delta 0,
    // disable_deblocking_filter_idc 1 (010); deblocked: idc 0 and both offsets se(0) (1 1 1), as many bits
    const uint32_t idc = l.deblock ? 7u : 2u;
    if (is_p)   // first_mb_in_slice 0, slice_type 5, pps 0, frame_num, three flags 0, slice_qp_delta 0, idc
      put_bits(raw, 0, 0x4Du << 11 | (uint32_t)meta[2] << 7 | 0x08u | idc, P_HEADER_BITS);   // 1 00110 1 ffff 0 0 0 1 010
    else
      put_bits(raw, 0, 0x222088u | idc, HEADER_BITS);  // 1 0001000 1 0000 010 0 0 1 010
    put_bits(raw, total, 1, 1);                  // rbsp_stop_one_bit
    reinterpret_cast<int*>(base + l.meta)[0] = nbytes;
  }
}

// ---- bit writing -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) h264_write_kernel(uint8_t* scratch, Layout l) {
  const int f = blockIdx.y, lane = threadIdx.x & 31;
  const int mb = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (mb >= l.nmb) return;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  uint32_t* raw = reinterpret_cast<uint32_t*>(base + l.raw);
  const int info = reinterpret_cast<const int*>(base + l.info)[mb];
  const bool is_p = frame_meta(scratch, l, f)[1] != 0;
  uint32_t pos = (uint32_t)reinterpret_cast<const int*>(base + l.off)[mb];
  const int mx = mb % l.wm, my = mb / l.wm;
  if (is_p) {   // mb_skip_run before a coded macroblock; the trailing run on a skipped last one
    const int skipped = (info >> 13) & 1;
    if (skipped && mb != l.nmb - 1) return;
    const int r = reinterpret_cast<const int*>(base + l.run)[mb];
    if (lane == 0) put_bits(raw, pos, r + 1, ue_bits(r));
    if (skipped) return;
    pos += ue_bits(r);
  }
  if ((info >> 7) & 1) {   // I_PCM: ue(25) (ue(30) in a P slice), alignment, 256 Y + 64 Cb + 64 Cr samples
    if (lane == 0) put_bits(raw, pos, is_p ? 31 : 26, 9);
    const uint32_t p0 = (pos + 9 + 7) & ~7u;
    const Planes rec(base + l.rec, l);
    for (int i = lane; i < 384; i += 32) {
      int v;
      if (i < 256) v = rec.y[(16 * my + (i >> 4)) * rec.ys + 16 * mx + (i & 15)];
      else {
        const int p = (i - 256) / 64, j = (i - 256) % 64;
        v = rec.chroma(p)[(8 * my + (j >> 3)) * rec.cs + 8 * mx + (j & 7)];
      }
      put_bits(raw, p0 + 8 * i, (uint32_t)v, 8);
    }
    return;
  }
  const bool inter = (info >> 8) & 1, nxn = (info >> 14) & 1;
  const uint8_t* tot = base + l.tot;
  int c[16], plane = 0, x = 0, y = 0, maxn = 0, nc = 0, n = 0;
  const bool present = lane < BLOCKS && block_present(lane, info);
  if (present) {
    block_geom(lane, mx, my, plane, x, y, maxn);
    if ((inter || nxn) && lane >= 1 && lane <= 16) maxn = 16;
    const int16_t* lev = reinterpret_cast<const int16_t*>(base + l.lev) + ((int64_t)mb * BLOCKS + lane) * 16;
    for (int k = 0; k < 16; k++) c[k] = k < maxn ? lev[k] : 0;
    nc = plane < 0 ? -1 : nc_of(tot, l, plane, x, y);
    BitSink sink{nullptr, 0, 0};
    n = cavlc_block(c, maxn, nc, sink);
  }
  int incl = n;
  for (int s = 1; s < 32; s <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, s);
    if (lane >= s) incl += v;
  }
  int hb = mb_header_bits(info, is_p);
  if (inter) {
    const int v = reinterpret_cast<const int*>(base + l.mvd)[mb];
    const int dx = (int16_t)(v & 0xffff), dy = v >> 16;
    const int cbp = inter_cbp(info), code = c_inter_cbp[cbp];
    hb += se_bits(dx) + se_bits(dy);
    if (lane == 0) {
      BitSink h{raw, pos, 0};
      h.u(1, 1);                                 // mb_type P_L0_16x16
      h.u(dx > 0 ? 2 * dx : -2 * dx + 1, se_bits(dx));
      h.u(dy > 0 ? 2 * dy : -2 * dy + 1, se_bits(dy));
      h.u(code + 1, ue_bits(code));
      if (cbp) h.u(1, 1);                        // mb_qp_delta 0
    }
  } else if (nxn) {
    const int* infos = reinterpret_cast<const int*>(base + l.info);
    const uint64_t* modes = reinterpret_cast<const uint64_t*>(base + l.modes);
    BitSink h{lane == 0 ? raw : nullptr, pos, 0};
    hb = i4_header(infos, modes, l.wm, mx, my, is_p, h);
  } else if (lane == 0) {
    const int mbt = i16_mb_type(info, is_p), cmode = (info >> 2) & 3;
    BitSink h{raw, pos, 0};
    h.u(mbt + 1, ue_bits(mbt));
    h.u(cmode + 1, ue_bits(cmode));
    h.u(1, 1);                                   // mb_qp_delta 0
  }
  if (present) {
    BitSink sink{raw, pos + hb + incl - n, 0};
    cavlc_block(c, maxn, nc, sink);
  }
}

// ---- emulation prevention and packing ----------------------------------------------------------------------------
// Per piece and start state z (0, 1, >= 2 zero bytes before it): ep[j] = {count(z=0), count(1), count(2),
// end states (2 bits each) | start state << 8 (written by the plan)}; the plan then overwrites count(0) with the
// piece's output offset.
__global__ void __launch_bounds__(128) h264_ep_count_kernel(uint8_t* scratch, Layout l) {
  const int f = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const int nbytes = reinterpret_cast<const int*>(base + l.meta)[0];
  const int lo = j * EP_PIECE;
  if (lo >= nbytes) return;
  const int hi = min(lo + EP_PIECE, nbytes);
  const uint8_t* raw = base + l.raw;
  int z[3] = {0, 1, 2}, cnt[3] = {0, 0, 0};
  for (int i = lo; i < hi; i++) {
    const int b = raw[i];
    for (int s = 0; s < 3; s++) {
      if (z[s] >= 2 && b <= 3) { cnt[s]++; z[s] = 0; }
      z[s] = b == 0 ? min(z[s] + 1, 2) : 0;
    }
  }
  int4* ep = reinterpret_cast<int4*>(base + l.ep);
  ep[j] = make_int4(cnt[0], cnt[1], cnt[2], z[0] | z[1] << 2 | z[2] << 4);
}

__global__ void __launch_bounds__(32) h264_ep_plan_kernel(uint8_t* scratch, Layout l, uint8_t* out, int64_t out_stride,
                                                          int64_t* out_len) {
  const int f = blockIdx.x, lane = threadIdx.x;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const int nbytes = reinterpret_cast<const int*>(base + l.meta)[0];
  const int np = (nbytes + EP_PIECE - 1) / EP_PIECE;
  int4* ep = reinterpret_cast<int4*>(base + l.ep);
  int state = 0, added = 0;                      // the NAL header byte 0x65 is not zero
  for (int j0 = 0; j0 < np; j0 += 32) {
    const int j = j0 + lane;
    const int4 e = j < np ? ep[j] : make_int4(0, 0, 0, 0);
    for (int k = 0; k < 32 && j0 + k < np; k++) {
      const int c0 = __shfl_sync(0xffffffffu, e.x, k), c1 = __shfl_sync(0xffffffffu, e.y, k);
      const int c2 = __shfl_sync(0xffffffffu, e.z, k), st = __shfl_sync(0xffffffffu, e.w, k);
      if (lane == k) ep[j] = make_int4((j0 + k) * EP_PIECE + added, 0, 0, state);
      added += state == 0 ? c0 : state == 1 ? c1 : c2;
      state = (st >> (2 * state)) & 3;
    }
  }
  if (lane == 0) {
    const int64_t body = 1 + (int64_t)nbytes + added;
    uint8_t* o = out + (int64_t)f * out_stride;
    o[0] = (uint8_t)(body >> 24); o[1] = (uint8_t)(body >> 16); o[2] = (uint8_t)(body >> 8); o[3] = (uint8_t)body;
    o[4] = frame_meta(scratch, l, f)[1] ? 0x61 : 0x65;   // nal_ref_idc 3, nal_unit_type 1 (P) or 5 (IDR slice)
    out_len[f] = 4 + body;
  }
}

__global__ void __launch_bounds__(128) h264_ep_emit_kernel(uint8_t* scratch, Layout l, uint8_t* out,
                                                           int64_t out_stride) {
  const int f = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  uint8_t* base = scratch + (int64_t)f * l.stride;
  const int nbytes = reinterpret_cast<const int*>(base + l.meta)[0];
  const int lo = j * EP_PIECE;
  if (lo >= nbytes) return;
  const int hi = min(lo + EP_PIECE, nbytes);
  const int4 e = reinterpret_cast<const int4*>(base + l.ep)[j];
  const uint8_t* raw = base + l.raw;
  uint8_t* o = out + (int64_t)f * out_stride + 5 + e.x;
  int z = e.w;
  for (int i = lo; i < hi; i++) {
    const int b = raw[i];
    if (z >= 2 && b <= 3) { *o++ = 3; z = 0; }
    *o++ = (uint8_t)b;
    z = b == 0 ? min(z + 1, 2) : 0;
  }
}

// ---- stream state -------------------------------------------------------------------------------------------------
// State: the stream position (int64) at byte 0, the previous picture's padded reconstruction (the Planes layout) from
// byte 256.  Frame f of a batch is stream position pos + f: an IDR picture when that is a multiple of gop, else a P
// picture with frame_num (position - last IDR) mod 16.
__global__ void __launch_bounds__(256) h264_frame_kernel(uint8_t* scratch, Layout l, const uint8_t* state, int gop,
                                                         int frames) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= frames) return;
  const int64_t n = (state ? *reinterpret_cast<const int64_t*>(state) : 0) + f;
  int* meta = reinterpret_cast<int*>(scratch + (int64_t)f * l.stride + l.meta);
  meta[1] = gop > 1 && n % gop != 0;
  meta[2] = (int)((n % gop) % 16);
}

// The last frame's reconstruction (deblocked when the stream is) becomes the state's picture, and the position advances by the batch.
__global__ void __launch_bounds__(256) h264_state_kernel(const uint8_t* scratch, Layout l, uint8_t* state,
                                                         int frames) {
  const uint4* src = reinterpret_cast<const uint4*>(scratch + (int64_t)(frames - 1) * l.stride + l.flt);
  uint4* dst = reinterpret_cast<uint4*>(state + 256);
  const int64_t n = (int64_t)l.nmb * 384 / 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = src[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<int64_t*>(state) += frames;
}

// ---- host: level, parameter sets ---------------------------------------------------------------------------------
struct LevelRow {
  int idc, mbps, fs;
};
const LevelRow kLevels[] = {{10, 1485, 99},      {11, 3000, 396},     {12, 6000, 396},     {13, 11880, 396},
                            {20, 11880, 396},    {21, 19800, 792},    {22, 20250, 1620},   {30, 40500, 1620},
                            {31, 108000, 3600},  {32, 216000, 5120},  {40, 245760, 8192},  {41, 245760, 8192},
                            {42, 522240, 8704},  {50, 589824, 22080}, {51, 983040, 36864}, {52, 2073600, 36864}};

bool fits(int wm, int hm, int fs) { return (int64_t)wm * hm <= fs && (int64_t)wm * wm <= 8 * fs && (int64_t)hm * hm <= 8 * fs; }

struct HostBits {
  std::vector<uint8_t> bytes;
  int n = 0;
  void u(uint64_t v, int len) {
    for (int i = len - 1; i >= 0; i--) {
      if (n % 8 == 0) bytes.push_back(0);
      if ((v >> i) & 1) bytes.back() |= (uint8_t)(0x80 >> (n % 8));
      n++;
    }
  }
  void ue(uint32_t v) {
    const uint64_t x = (uint64_t)v + 1;
    int L = 0;
    while ((x >> L) > 1) L++;
    u(x, 2 * L + 1);
  }
  void se(int v) { ue(v > 0 ? 2 * v - 1 : -2 * v); }
  std::vector<uint8_t> nal(int type) {   // trailing bits, emulation prevention, the header byte
    u(1, 1);
    while (n % 8) u(0, 1);
    std::vector<uint8_t> o{(uint8_t)(0x60 | type)};
    int zeros = 0;
    for (uint8_t b : bytes) {
      if (zeros >= 2 && b <= 3) { o.push_back(3); zeros = 0; }
      o.push_back(b);
      zeros = b == 0 ? zeros + 1 : 0;
    }
    return o;
  }
};

}  // namespace

int h264_level_idc(int W, int H, int fps_num, int fps_den) {
  const int wm = (W + 15) / 16, hm = (H + 15) / 16;
  for (const LevelRow& r : kLevels)
    if (fits(wm, hm, r.fs) && (int64_t)wm * hm * fps_num <= (int64_t)r.mbps * fps_den) return r.idc;
  return fits(wm, hm, MAX_MBS) ? 52 : -1;
}

int64_t h264_bound(int W, int H) {
  if (W <= 0 || H <= 0 || (W & 1) || (H & 1) || W > 65536 || H > 65536) return -1;
  if (h264_level_idc(W, H, 0, 1) < 0) return -1;
  const int64_t n = raw_bytes_bound(((W + 15) / 16) * ((H + 15) / 16));
  return 5 + n + (n + 1) / 2;
}

int64_t h264_p_bound(int W, int H) {
  if (h264_bound(W, H) < 0) return -1;
  const int64_t n = raw_bytes_bound_p(((W + 15) / 16) * ((H + 15) / 16));
  return 5 + n + (n + 1) / 2;
}

size_t h264_state_bytes(int H, int W) {
  if (h264_bound(W, H) < 0) return 0;
  return (size_t)(256 + align256((int64_t)((W + 15) / 16) * ((H + 15) / 16) * 384));
}

size_t h264_scratch_bytes(int64_t frames, int H, int W, bool deblock, bool intra4x4) {
  if (frames <= 0 || frames > 65535 || h264_bound(W, H) < 0) return 0;
  return (size_t)(frames * layout(H, W, deblock, intra4x4).stride);
}

int32_t h264_parameter_sets(int W, int H, int qp, int fps_num, int fps_den, int gop, uint8_t* out, int64_t cap) {
  if (h264_bound(W, H) < 0 || qp < 0 || qp > 51 || fps_num <= 0 || fps_den <= 0 || fps_num > (INT32_MAX / 2)) return -1;
  if (gop < 1 || gop > 65535) return -1;
  const int wc = (W + 15) / 16 * 16, hc = (H + 15) / 16 * 16;
  HostBits s;
  s.u(66, 8);                    // profile_idc: Baseline
  s.u(0xC0, 8);                  // constraint_set0_flag, constraint_set1_flag: Constrained Baseline
  s.u(h264_level_idc(W, H, fps_num, fps_den), 8);
  s.ue(0);                       // seq_parameter_set_id
  s.ue(0);                       // log2_max_frame_num_minus4
  s.ue(2);                       // pic_order_cnt_type
  s.ue(gop > 1 ? 1 : 0);         // max_num_ref_frames: a P picture refers to the previous picture
  s.u(0, 1);                     // gaps_in_frame_num_value_allowed_flag
  s.ue(wc / 16 - 1);
  s.ue(hc / 16 - 1);
  s.u(1, 1);                     // frame_mbs_only_flag
  s.u(1, 1);                     // direct_8x8_inference_flag
  const bool crop = wc != W || hc != H;
  s.u(crop, 1);
  if (crop) {
    s.ue(0);
    s.ue((wc - W) / 2);
    s.ue(0);
    s.ue((hc - H) / 2);
  }
  s.u(1, 1);                     // vui_parameters_present_flag
  s.u(0, 1);                     // aspect_ratio_info_present_flag
  s.u(0, 1);                     // overscan_info_present_flag
  s.u(1, 1);                     // video_signal_type_present_flag
  s.u(5, 3);                     // video_format: unspecified
  s.u(0, 1);                     // video_full_range_flag: limited range
  s.u(1, 1);                     // colour_description_present_flag
  s.u(2, 8);                     // colour_primaries: unspecified
  s.u(2, 8);                     // transfer_characteristics: unspecified
  s.u(6, 8);                     // matrix_coefficients: BT.601
  s.u(0, 1);                     // chroma_loc_info_present_flag
  s.u(1, 1);                     // timing_info_present_flag
  s.u((uint32_t)fps_den, 32);    // num_units_in_tick
  s.u(2 * (uint32_t)fps_num, 32);// time_scale
  s.u(1, 1);                     // fixed_frame_rate_flag
  s.u(0, 1);                     // nal_hrd_parameters_present_flag
  s.u(0, 1);                     // vcl_hrd_parameters_present_flag
  s.u(0, 1);                     // pic_struct_present_flag
  s.u(0, 1);                     // bitstream_restriction_flag
  const std::vector<uint8_t> sps = s.nal(7);
  HostBits p;
  p.ue(0);                       // pic_parameter_set_id
  p.ue(0);                       // seq_parameter_set_id
  p.u(0, 1);                     // entropy_coding_mode_flag: CAVLC
  p.u(0, 1);                     // bottom_field_pic_order_in_frame_present_flag
  p.ue(0);                       // num_slice_groups_minus1
  p.ue(0);
  p.ue(0);                       // num_ref_idx_l0/l1_default_active_minus1
  p.u(0, 1);                     // weighted_pred_flag
  p.u(0, 2);                     // weighted_bipred_idc
  p.se(qp - 26);                 // pic_init_qp_minus26
  p.se(0);                       // pic_init_qs_minus26
  p.se(0);                       // chroma_qp_index_offset
  p.u(1, 1);                     // deblocking_filter_control_present_flag
  p.u(0, 1);                     // constrained_intra_pred_flag
  p.u(0, 1);                     // redundant_pic_cnt_present_flag
  const std::vector<uint8_t> pps = p.nal(8);
  const int64_t need = 4 + (int64_t)sps.size() + (int64_t)pps.size();
  if (out == nullptr || cap < need) return -1;
  int64_t o = 0;
  for (const std::vector<uint8_t>* v : {&sps, &pps}) {
    out[o++] = (uint8_t)(v->size() >> 8);
    out[o++] = (uint8_t)v->size();
    for (uint8_t b : *v) out[o++] = b;
  }
  return (int32_t)need;
}

void launch_h264_encode(int frames, int H, int W, int qp, int gop, bool deblock, bool intra4x4, const uint8_t* rgb,
                        uint8_t* state, void* scratch, uint8_t* out, int64_t out_stride, int64_t* out_len,
                        cudaStream_t stream) {
  const Layout l = layout(H, W, deblock, intra4x4);
  uint8_t* s = static_cast<uint8_t*>(scratch);
  const unsigned F = (unsigned)frames;
  h264_convert_kernel<<<dim3((unsigned)((64 * l.nmb + 255) / 256), F), 256, 0, stream>>>(rgb, s, l);
  count_launch();
  h264_frame_kernel<<<(F + 255) / 256, 256, 0, stream>>>(s, l, state, gop, frames);
  count_launch();
  // The wavefront over (frame, line): step k encodes line k - lag f of every frame f that has one (anti-diagonals
  // mbx + mby, or lines mbx + 2 mby in a deblocked P stream) and then filters line k - lag f - DB_LAG.
  const int slope = deblock && gop > 1 ? 2 : 1, D = l.wm + slope * (l.hm - 1), DB = l.wm + 2 * (l.hm - 1);
  const int lag = gop > 1 ? (deblock ? LAG_DB : LAG) : 0;
  auto line_len = [&](int d, int sl) {
    if (d < 0 || d >= l.wm + sl * (l.hm - 1)) return 0;
    return sl == 1 ? std::min(d, l.wm - 1) - std::max(0, d - l.hm + 1) + 1
                   : std::min(d / 2, l.hm - 1) - std::max(0, (d - l.wm + 2) / 2) + 1;
  };
  // the frames with a line at step k of a wavefront `off` steps behind, `lines` lines long, and its longest line
  auto frames_at = [&](int k, int off, int lines, int sl, int& f_lo, int& f_hi) {
    f_lo = lag ? std::max(0, (k - off - (lines - 1) + lag - 1) / lag) : 0;
    f_hi = lag ? std::min(frames - 1, (k - off) / lag) : frames - 1;
    int n = 0;   // 0 when lag > lines leaves a step between two frames' wavefronts
    for (int f = f_lo; f <= f_hi && n < std::min(l.wm, l.hm); f++) n = std::max(n, line_len(k - off - lag * f, sl));
    return n;
  };
  const int steps = std::max(D, deblock ? DB + DB_LAG : 0) + (frames - 1) * lag;
  for (int k = 0; k < steps; k++) {
    int f_lo, f_hi;
    int n = frames_at(k, 0, D, slope, f_lo, f_hi);
    if (n > 0) {
      const dim3 grid((unsigned)n, (unsigned)(f_hi - f_lo + 1));
      if (intra4x4) h264_mb_kernel<true><<<grid, 128, 0, stream>>>(k, lag, slope, f_lo, qp, s, state, l);
      else h264_mb_kernel<false><<<grid, 128, 0, stream>>>(k, lag, slope, f_lo, qp, s, state, l);
      count_launch();
    }
    if (!deblock) continue;
    n = frames_at(k, DB_LAG, DB, 2, f_lo, f_hi);
    if (n > 0) {
      h264_deblock_kernel<<<dim3((unsigned)n, (unsigned)(f_hi - f_lo + 1)), 32, 0, stream>>>(k, lag, f_lo, qp, s, l);
      count_launch();
    }
  }
  const unsigned mbb = (unsigned)((l.nmb + 127) / 128);
  if (gop > 1) {
    h264_mvp_kernel<<<dim3(mbb, F), 128, 0, stream>>>(s, l);
    count_launch();
    h264_run_kernel<<<dim3(mbb, F), 128, 0, stream>>>(s, l);
    count_launch();
  }
  h264_scan_kernel<<<F, 1024, 0, stream>>>(s, l);
  count_launch();
  h264_write_kernel<<<dim3((unsigned)((l.nmb + 3) / 4), F), 128, 0, stream>>>(s, l);
  count_launch();
  const unsigned pb = (unsigned)((l.pieces + 127) / 128);
  h264_ep_count_kernel<<<dim3(pb, F), 128, 0, stream>>>(s, l);
  count_launch();
  h264_ep_plan_kernel<<<F, 32, 0, stream>>>(s, l, out, out_stride, out_len);
  count_launch();
  h264_ep_emit_kernel<<<dim3(pb, F), 128, 0, stream>>>(s, l, out, out_stride);
  count_launch();
  if (state) {
    h264_state_kernel<<<std::min(1024u, (unsigned)((l.nmb * 24 + 255) / 256)), 256, 0, stream>>>(s, l, state, frames);
    count_launch();
  }
}

}  // namespace gab
