// Internal launcher declarations + small device helpers shared by the .cu files.
#pragma once
#include "common.cuh"

namespace gab {

// SH constants (values of utils/sh_utils.py:26-43)
#define SH_C0 0.28209479177387814f
#define SH_C1 0.4886025119029199f
#define SH_C2_0 1.0925484305920792f
#define SH_C2_1 -1.0925484305920792f
#define SH_C2_2 0.31539156525252005f
#define SH_C2_3 -1.0925484305920792f
#define SH_C2_4 0.5462742152960396f
#define SH_C3_0 -0.5900435899266435f
#define SH_C3_1 2.890611442640554f
#define SH_C3_2 -0.4570457994644658f
#define SH_C3_3 0.3731763325901154f
#define SH_C3_4 -0.4570457994644658f
#define SH_C3_5 1.445305721320277f
#define SH_C3_6 -0.5900435899266435f

void count_launch();
int tune_get(int knob);  // api.cu: current value of a gab200_tune() knob

// Programmatic dependent launch (sm_90).  A kernel launched through launch_pdl may start while the kernel before it on
// the stream is still draining (stream capture turns this into a programmatic graph edge), so its launch and the
// CTAs' start-up overlap the predecessor's tail.  Every such kernel calls pdl_wait() in every CTA before it reads or
// writes global memory -- it returns once the predecessor grid has completed and its writes are visible, and since
// the predecessor waited the same way, once every earlier kernel has -- and then pdl_trigger(), which lets the next
// kernel launch once all of this grid's CTAs have been scheduled.  Both are no-ops in a kernel launched without the
// attribute.  Only kernel parameters and shared memory are touched above the wait: the camera, bg and dL/dimage may
// be written by a kernel just before (a loss kernel, a torch copy), so they are read after it like everything else.
template <typename... Params, typename... Args>
void launch_pdl(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  const cudaLaunchConfig_t cfg = {grid, block, smem, stream, &attr, 1};
  cudaLaunchKernelEx(&cfg, kernel, static_cast<Args&&>(args)...);
  count_launch();
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Exact per-tile-row span of the region where a splat can reach alpha >= 1/255:
//   q(d) = 1/2 (A dx^2 + C dy^2) + B dx dy <= ln(255 * opacity)          (the blend's own accept test)
// For tile row ty the pixel centres have dy in [16 ty - py, 16 ty + 15 - py]; the x-extent of the ellipse over
// that band is closed-form (extreme point if it lies in the band, else the better band edge).  The span is
// intersected with the reference's 3-sigma bounding-square columns [rx0, rx1) so the emitted instance list is
// always a SUBSEQUENCE of the reference's.  Margins: +0.01 in the exponent (alpha down to 0.99/255 kept) and
// +-0.02 px, i.e. only pairs that contribute exactly nothing are dropped.
struct TileSpan {
  bool any, full;
  float px, py, A, B, tau2A, det, dxmax, ystar, ymax;
  int rx0, rx1;
  __device__ __forceinline__ TileSpan(float px_, float py_, float A_, float B_, float C_, float opacity, int rx0_,
                                      int rx1_)
      : px(px_), py(py_), A(A_), B(B_), rx0(rx0_), rx1(rx1_) {
    const float tau = logf(255.f * opacity) + 0.01f;
    det = A_ * C_ - B_ * B_;
    const bool pd = (det > 0.f) && (A_ > 0.f) && (C_ > 0.f) && (det < 3.0e38f);
    any = tau > 0.f;
    full = !pd || !(tau < 3.0e38f);
    const float tau2 = 2.f * tau;
    tau2A = tau2 * A_;
    dxmax = sqrtf(fmaxf(0.f, tau2 * C_ / det));
    ymax = sqrtf(fmaxf(0.f, tau2 * A_ / det));
    ystar = (B_ / C_) * dxmax;
  }
  __device__ __forceinline__ float half_width(float dy) const { return sqrtf(fmaxf(0.f, tau2A - det * dy * dy)); }
  __device__ __forceinline__ void row(int ty, int& cx0, int& cx1) const {
    if (!any) { cx0 = cx1 = rx0; return; }
    if (full) { cx0 = rx0; cx1 = rx1; return; }
    const float a = (float)(ty * GAB_TILE) - py, b = a + (float)(GAB_TILE - 1);
    const float lo = fmaxf(a, -ymax) - 0.02f, hi = fminf(b, ymax) + 0.02f;
    if (lo > hi) { cx0 = cx1 = rx0; return; }
    float xr, xl;
    const float hl = half_width(lo), hh = half_width(hi);
    if (-ystar >= lo && -ystar <= hi) xr = dxmax;
    else xr = fmaxf((-B * lo + hl) / A, (-B * hi + hh) / A);
    if (ystar >= lo && ystar <= hi) xl = -dxmax;
    else xl = fminf((-B * lo - hl) / A, (-B * hi - hh) / A);
    const float X0 = px + xl - 0.02f, X1 = px + xr + 0.02f;
    int t0 = (int)ceilf((X0 - (float)(GAB_TILE - 1)) * (1.0f / GAB_TILE));
    int t1 = (int)floorf(X1 * (1.0f / GAB_TILE)) + 1;
    cx0 = min(max(t0, rx0), rx1);
    cx1 = max(min(t1, rx1), cx0);
  }
};

// ---- launchers (each counts its launches) ----
// Per-splat depth sort as a bucket sort (binning.cu header): bookkeeping arrays in the geometry buffer.
#define GAB_DEPTH_BUCKET_CAP 2048   // splats one bucket may hold before the frame falls back to the radix path
// the frame counters of the public header (GAB200_CTR_*) + two private words: the 64-bit instance total
// (meta[GAB_META_TOTAL64 .. +1], 8-byte aligned), from which GAB200_CTR_NUM_RENDERED_HI is published
#define GAB_DEPTH_META_WORDS (GAB200_NUM_COUNTERS + 2)
#define GAB_META_TOTAL64 GAB200_NUM_COUNTERS
struct DepthBuckets {
  uint32_t* counts;     // [nb] splats per bucket           } zeroed together with meta before preprocess
  uint32_t* tiles;      // [nb] instances per bucket        }
  uint32_t* meta;       // [GAB_DEPTH_META_WORDS]           }
  uint32_t* start;      // [nb] exclusive prefix of counts
  uint32_t* tile_base;  // [nb] exclusive prefix of tiles
  uint32_t* rank;       // [P]  arrival rank of the splat inside its bucket
  uint32_t nb;          // buckets (power of two)
  uint32_t lo, hi;      // hinted key range; keys outside are clamped to the end buckets (order is preserved)
  float scale;          // nb / (hi - lo + 1)
  int enabled;          // 0: only meta[0..1] (min/max key) are maintained
};
// Monotonic non-decreasing in `key` (u32->f32 conversion, multiply by a positive constant and truncation all are),
// which is all the bucket sort needs.  Evaluated in preprocess.cu only (one translation unit, one set of flags).
__device__ __forceinline__ uint32_t depth_bucket(uint32_t key, const DepthBuckets& d) {
  if (key <= d.lo) return 0u;
  if (key >= d.hi) return d.nb - 1u;
  const uint32_t b = (uint32_t)(__uint2float_rz(key - d.lo) * d.scale);
  return b < d.nb ? b : d.nb - 1u;
}
// cameras == NULL: the camera of `a`, its field of view from the device float[2] `tanfov`
// (gab200_forward_device_fov) or, when that is NULL, a.tanfovx / tanfovy.  Otherwise `views` cameras
// (gab200_forward_views*): grid (splat blocks, views); camera row k of `cameras` renders virtual splats k * P + i
// (rec / aux / tiles / depth keys / ids / radii / visibility / clamp bits), tile counts at k * (gx * gy) + the tile
// in the view.  clamped != nullptr: also the colour clamp bits (the backward reads them); tile_count != nullptr: also
// count the instances of every tile (counting tile sort, tile_sort.cu); rec_depth: the records carry the view-space
// depth in q2.w (the depth_alpha forms)
void launch_preprocess(const gab200_forward_args& a, int views, const float* cameras, const float* tanfov,
                       SplatRec* rec, SplatAux* aux, uint32_t* tiles_touched, uint8_t* clamped, uint32_t* depth_keys,
                       uint32_t* ids, const DepthBuckets& buckets, uint32_t* tile_count, bool rec_depth,
                       cudaStream_t stream);
// depth_keys [P] (by splat) -> sorted_ids [M] in (key, id) order and offsets [M] = inclusive instance counts
// also publishes the frame counters (capacity, seq, overflow) of the bucket-sorted frame
void launch_depth_bucket_sort(int P, const DepthBuckets& buckets, const uint32_t* depth_keys,
                              const uint32_t* tiles_touched, uint32_t* scratch_keys, uint32_t* sorted_ids,
                              uint32_t* offsets, uint32_t capacity, uint32_t seq, uint32_t* sticky_overflow,
                              cudaStream_t stream);
void launch_bind_activate(const gab200_forward_args& a, float* means3D, float* opacities, float* scales, float* cov3D,
                          cudaStream_t stream);
void launch_mark_visible(int P, const float* means3D, const float* V, uint8_t* present, cudaStream_t stream);
// counters[NUM_LISTED] (+ NUM_RENDERED from offsets when given) of a radix-sorted frame (P > 0; pass 0 for a
// bucket-sorted one, whose kernels wrote them), capacity and sequence number
void launch_publish_counters(uint32_t* counters, const uint32_t* offsets, int P, uint32_t capacity, uint32_t seq,
                             uint32_t* sticky_overflow, cudaStream_t stream);
// Buffers the emission grid clears before the tile sort (preprocess.cu emit_clears); zero / null: nothing to clear
struct EmitClears {
  bool sentinel = false;      // keys past the device count up to the capacity get the sentinel 0xffffffff
  uint8_t* mask = nullptr;    // block masks [0, n_mask) zeroed
  uint32_t n_mask = 0;
  uint2* ranges = nullptr;    // tile ranges [0, n_ranges) zeroed
  uint32_t n_ranges = 0;
};
// `capacity`: instances the key/value arrays hold -- anything beyond is dropped (the frame's counters say so);
// counters[BUCKET_OVERFLOW] != 0 (depth order unusable) emits nothing.
void launch_emit_keys(int P, int gx, int gy, const SplatRec* rec, const SplatAux* aux, const uint32_t* order,
                      const uint32_t* offsets, const uint32_t* order_count, const uint32_t* counters, uint32_t capacity,
                      uint32_t* cursor, uint32_t* keys, uint32_t* vals, int exact_binning, const EmitClears& clr,
                      cudaStream_t stream);
// the same over the P virtual splats of a multi-view frame, view_splats per view: instances of virtual splat v go to
// the tiles (v / view_splats) * (gx * gy) + the tile in the view
void launch_emit_keys_views(int P, int gx, int gy, const SplatRec* rec, const SplatAux* aux, const uint32_t* order,
                            const uint32_t* offsets, const uint32_t* order_count, const uint32_t* counters, uint32_t cap,
                            uint32_t* cursor, uint32_t* keys, uint32_t* vals, int exact_binning, int view_splats,
                            const EmitClears& clr, cudaStream_t stream);
// keys[0..N) sorted; entries with key >= tiles are padding (sentinel) behind the last real instance
void launch_tile_ranges(int64_t N, uint32_t tiles, const uint32_t* keys, uint2* ranges, cudaStream_t stream);
void launch_expand_keys(int64_t N, const uint32_t* tile_keys, const uint32_t* ids, const SplatAux* aux, uint64_t* out,
                        cudaStream_t stream);
// tile_sort.cu
#define GAB_TILE_SORT_SMEM 2048  // entries one CTA sorts in shared memory; longer tile lists take the bitmap kernel
// tile_count != nullptr: ranges / cursors / counters[NUM_RENDERED] from the per-tile counts (ranges cut at `clamp`);
// always: heaviest-first tile order + heavy/light split points (order_info[0..1]) + number of long tiles ([2])
void launch_tile_scan_order(int tiles, const uint32_t* tile_count, uint32_t clamp, uint2* ranges, uint32_t* cursor,
                            uint32_t* order, uint32_t* order_info, uint32_t* counters, int heavy_fwd, int heavy_bwd,
                            cudaStream_t stream);
// every tile's (rank, id) segment sorted by rank; ids written back in place
void launch_tile_sort(int tiles, const uint2* ranges, const uint32_t* order, const uint32_t* order_info, uint32_t* keys,
                      uint32_t* vals, const uint32_t* rank_to_id, const uint32_t* listed, int P, cudaStream_t stream);
void launch_expand_keys_by_range(int tiles, const uint2* ranges, const uint32_t* ids, const SplatAux* aux, uint64_t* out,
                                 cudaStream_t stream);

// binning.cu (cub)
size_t scan_temp_bytes(int P);
cudaError_t run_scan(void* temp, size_t temp_bytes, const uint32_t* order, const uint32_t* tiles_touched, uint32_t* out,
                     int P, cudaStream_t stream);
size_t sort_temp_bytes(int64_t N, int end_bit);
cudaError_t run_sort(void* temp, size_t temp_bytes, uint32_t* keys_a, uint32_t* keys_b, uint32_t* vals_a,
                     uint32_t* vals_b, int64_t N, int end_bit, int* selector_out, cudaStream_t stream);

// blend.cu
// `views` images of one size (1: a single view): global tile g is tile g % (gx * gy) of view g / (gx * gy).
// out_color [views,3,H,W] / out_rgb8 [views,H,W,3]: either may be NULL.  final_T != NULL (the training forms): also
// final_T / n_contrib [views,H,W] and the per-instance block masks, kept for launch_blend_backward.
// out_alpha / out_depth [views,H,W]: the accumulated alpha and depth planes (either may be NULL; records with z in q2.w)
void launch_blend_forward(int views, int W, int H, const uint2* ranges, const uint32_t* order,
                          const uint32_t* order_info, const uint32_t* point_list, const SplatRec* rec, const float* bg,
                          float* out_color, float* final_T, uint32_t* n_contrib, uint8_t* strip_mask, uint8_t* out_rgb8,
                          float* out_alpha, float* out_depth, cudaStream_t stream);
// the same tiles: dL_dpix [views,3,H,W]; g2d rows of the views * P virtual splats.  da: also the plane gradients
// dL_dalpha / dL_ddepth [views,H,W] (NULL: zero); dL/dz -> g2d slot 9 of each virtual splat's row
void launch_blend_backward(int views, int W, int H, const uint2* ranges, const uint32_t* order,
                           const uint32_t* order_info, const uint32_t* point_list, const SplatRec* rec, const float* bg,
                           const float* final_T, const uint32_t* n_contrib, const float* dL_dpix,
                           const uint8_t* strip_mask, float* g2d, bool da, const float* dL_dalpha,
                           const float* dL_ddepth, cudaStream_t stream);
// preprocess_bwd.cu
// depth: g2d slot 9 holds dL/dz (gab200_backward_depth_alpha), added to dL/dmean through the view matrix's third row;
// no multicast
void launch_preprocess_backward(const gab200_backward_args& b, const SplatRec* rec, const SplatAux* aux,
                                const uint8_t* clamped, const float* g2d, float* face_scratch, const float* tanfov,
                                cudaStream_t stream, bool depth = false);
// gab200_backward_views (BOUND_RAW, no colors_precomp, no multicast): one thread per real splat sums the gradients of
// its `views` virtual splats (camera row k of `cameras`; rec / aux / clamped / g2d rows k * P + i) and stores each
// parameter gradient once; dL_dmeans2D [views,P,3]; face-frame gradients as launch_preprocess_backward's.
// depth: g2d slot 9 holds each virtual splat's dL/dz (gab200_backward_views_depth_alpha), added through view k's own
// view-matrix row
void launch_preprocess_backward_views(const gab200_backward_args& b, int views, const float* cameras,
                                      const SplatAux* aux, const uint8_t* clamped, const float* g2d,
                                      float* face_scratch, cudaStream_t stream, bool depth = false);
#define GAB_FACE_GRAD_STRIDE 13  // per-splat face-frame gradient record: centre 3, orientation 9, scale 1

// face_frame.cu
void launch_face_frame_forward(int F, const float* verts, const int32_t* faces, float* fc, float* fR, float* fs,
                               cudaStream_t stream);
void launch_face_frame_backward(int F, const float* verts, const int32_t* faces, const float* g_fc, const float* g_fR,
                                const float* g_fs, float* g_verts, cudaStream_t stream);

// loss.cu
void launch_l1_loss_u8(int64_t n, const float* img, const uint8_t* gt, const float* upstream, float* grad, float* loss,
                       cudaStream_t stream);

void launch_photometric_loss(int C, int H, int W, const float* img, const void* gt, int gt_is_u8, float lambda,
                             float* grad, float* loss, float* scratch, cudaStream_t stream);

// composite.cu
void launch_composite_rgba(int64_t views, int H, int W, const uint8_t* rgba, const float* bg, uint8_t* rgb,
                           uint8_t* mask, cudaStream_t stream);

// frames.cu
int frame_tiles(int H, int W);
void launch_frame_encode_plan(int64_t frames, int H, int W, const uint8_t* gt, const uint8_t* mask, uint32_t* units,
                              cudaStream_t stream);
void launch_frame_encode(int64_t frames, int H, int W, const uint8_t* gt, const uint8_t* mask,
                         const int64_t* frame_base, const uint32_t* tile_off, uint8_t* arena, cudaStream_t stream);
void launch_frame_decode(int views, int H, int W, const int32_t* ids, const uint8_t* arena, const int64_t* frame_base,
                         const uint32_t* tile_off, uint8_t* gt, uint8_t* mask, cudaStream_t stream);

// schedule.cu
void launch_schedule_sample(int records, int views, int length, const float* cams, const int32_t* timesteps,
                            const int32_t* frame_ids, const int32_t* order, const int32_t* cursor, float* cam_out,
                            int32_t* timestep_out, int32_t* ids_out, int32_t* rows_out, int32_t* exhausted,
                            cudaStream_t stream);
void launch_schedule_commit(int length, const int32_t* overflow_flag, const int32_t* exhausted, const float* loss,
                            float* losses, int32_t* cursor, cudaStream_t stream);

// metrics.cu
size_t metrics_scratch_bytes(int H, int W);
void launch_image_metrics(int H, int W, int kind, const void* render, const uint8_t* gt, const int32_t* row, int rows,
                          const int32_t* skip, float* table, void* scratch, cudaStream_t stream);

// lpips.cu
size_t lpips_weights_bytes(int net);
size_t lpips_scratch_bytes(int net, int H, int W);
size_t lpips_features_bytes(int net, int H, int W);
int lpips_conv_count(int net);
void launch_lpips_pack(int net, const float* const* conv_w, const float* const* conv_b, const float* const* lin,
                       float* packed, cudaStream_t stream);
void launch_lpips(const gab200_lpips_args& a, cudaStream_t stream);

// mesh.cu
size_t mesh_scratch_bytes(int F, int W, int H);
cudaError_t launch_mesh_render(const gab200_mesh_args& a, cudaStream_t stream);

// densify.cu
size_t densify_scratch_bytes(int P, int F);
cudaError_t launch_densify_plan(const gab200_densify_args& a, cudaStream_t stream);
cudaError_t launch_densify_apply(const gab200_densify_args& a, const gab200_densify_out& o, cudaStream_t stream);
void launch_densify_stats(int P, const float* vgrad, const int32_t* radii, float* accum, float* denom, float* max_radii,
                          const int32_t* skip, cudaStream_t stream);

// regularize.cu
cudaError_t launch_regularize_forward(const gab200_regularize_args& a, cudaStream_t stream);
cudaError_t launch_regularize_backward(const gab200_regularize_args& a, const float* g_out, cudaStream_t stream);

// nvls.cu
void launch_nvls_allreduce(float* mc, int64_t n, int rank, int world, cudaStream_t stream);

// flame.cu
size_t flame_scratch_bytes(int V, int n_expr);
void launch_flame_prepare(const gab200_flame_assets& a, const float* shape, const float* static_offset, void* scratch,
                          cudaStream_t stream);
void launch_flame_forward(const gab200_flame_frame_args& g, float* verts, float* verts_cano, cudaStream_t stream);
void launch_flame_backward(const gab200_flame_frame_args& g, const float* g_verts, const float* g_cano,
                           const gab200_flame_grads& grads, cudaStream_t stream);

// optim.cu
void launch_adam(int num_segments, const gab200_adam_segment* segs, int64_t step, double beta1, double beta2, double eps,
                 cudaStream_t stream);
void launch_adam_device(int num_segments, const gab200_adam_device_segment* segs, double beta1, double beta2,
                        double eps, const int32_t* skip, cudaStream_t stream);

}  // namespace gab
