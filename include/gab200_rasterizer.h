/*
 * gab200_rasterizer.h -- C ABI of the H100-native (sm_90a) differentiable Gaussian-splat rasterizer with fused
 * FLAME mesh binding (libgaussianavatars_b200.so).
 *
 * This is the drop-in boundary for the one native operator GaussianAvatars calls on its hot path:
 *   reference call site ........ gaussian_renderer/__init__.py:15,37-52,86-94
 *   reference native module .... diff_gaussian_rasterization._C (submodule graphdeco-inria/diff-gaussian-rasterization
 *                                @59f5f77, ABSENT from /root/reference; its pybind surface is
 *                                rasterize_gaussians / rasterize_gaussians_backward / mark_visible, SURVEY.md 2.2, 8a/a8-a9)
 * Each entry point below names the reference interface it replaces.
 *
 * Conventions
 *   - Every pointer is a DEVICE pointer owned by the caller unless stated otherwise; fp32 unless stated.
 *   - Matrices are the row-major flatten of the (4,4) tensors GaussianAvatars builds
 *     (world_view_transform = W2C^T, full_proj_transform = (P W2C)^T; scene/cameras.py:44-46).
 *   - Nothing a call leaves behind in the library affects a later result: what persists is a launch counter,
 *     the opt-in stage/host timers (atomics), the tuning knobs of gab200_tune(), and per host thread a 64-byte
 *     pinned read-back slot (hints such as binning_hint / depth_hint_* travel through the caller; the layout of
 *     the three scratch buffers is a pure function of the arguments).  Thread-safe per stream; no
 *     exceptions cross the ABI: functions return >= 0 on success and a negative gab200_status on failure
 *     (gab200_status_string() explains it).
 *   - Scratch memory is obtained through caller-supplied allocation callbacks, mirroring the reference
 *     module's three resizable byte buffers (geometry / binning / image; SURVEY.md 8a/a9).  The callbacks
 *     are invoked on the calling host thread, must return device memory aligned to 256 B that stays valid
 *     until the matching gab200_backward() has run (or is never called).
 */
#ifndef GAB200_RASTERIZER_H
#define GAB200_RASTERIZER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GAB200_ABI_VERSION 3

typedef enum gab200_status {
  GAB200_OK = 0,
  GAB200_ERR_INVALID_ARGUMENT = -1, /* bad shape / missing pointer / inconsistent option        */
  GAB200_ERR_CUDA = -2,             /* a CUDA runtime call or kernel failed (see cudaGetLastError) */
  GAB200_ERR_ALLOC = -3,            /* an allocation callback returned NULL                       */
  GAB200_ERR_ARCH = -4,             /* device is not compute capability 9.0 (sm_90a code only)   */
  GAB200_ERR_OVERFLOW = -5          /* more than 2^32-1 (splat,tile) instances                    */
} gab200_status;

/* Input interpretation. */
typedef enum gab200_input_mode {
  /* Reference surface: means3D world-space, scales already exp()-activated, rotations unit wxyz (used as given),
   * opacities already sigmoid()-activated -- exactly what render() passes today
   * (gaussian_renderer/__init__.py:54-94 <- scene/gaussian_model.py:113-160). */
  GAB200_INPUT_ACTIVATED = 0,
  /* Fused surface: the RAW parameters of GaussianModel (_xyz local, _scaling log, _rotation unnormalised,
   * _opacity logit, _features_dc/_features_rest) plus the per-face frame; the binding transform of
   * scene/gaussian_model.py:113-160 runs inside the preprocess kernel.  binding == NULL means identity frame. */
  GAB200_INPUT_BOUND_RAW = 1
} gab200_input_mode;

/* How gab200_forward learns N, the number of (splat,tile) instances of the frame (the reference copies it to the
 * host in the middle of every forward to size its binning buffer: rasterizer_impl.cu, SURVEY.md 2.4 K2 / 7.3). */
typedef enum gab200_sync_mode {
  /* One host wait in the MIDDLE of the forward (after preprocess + per-splat depth sort): the binning buffer is
   * sized for exactly N.  Needs no hint; this is what the first frame of a model uses. */
  GAB200_SYNC_EXACT = 0,
  /* binning_hint (> 0) is a hard CAPACITY: the whole forward is enqueued without waiting, then the host waits for
   * the frame counters at the END of the call (they were written long before in the common case) and, only if the
   * frame needed more than the capacity or the depth-bucket hint did not fit, re-enqueues the affected stages with
   * the exact size.  The result is the same as GAB200_SYNC_EXACT's, bit for bit; the GPU never idles behind the host. */
  GAB200_SYNC_LATE = 1,
  /* Never waits (required while the stream is being captured into a CUDA graph).  The frame counters are copied
   * to `counters_host`; the caller inspects them whenever it likes (gab200_counters_ok()).  A frame that overflowed
   * its capacity was rendered from a truncated instance list (memory-safe, wrong image): redo it with a larger
   * binning_hint. */
  GAB200_SYNC_NONE = 2
} gab200_sync_mode;

/* Frame counters (device: gab200_frame_state.device_counters; host copy: counters_host), 8 x uint32. */
enum {
  GAB200_CTR_NOT_MIN_DEPTH_KEY = 0, /* ~(smallest depth key among the splats that emitted instances) */
  GAB200_CTR_MAX_DEPTH_KEY = 1,
  GAB200_CTR_NUM_RENDERED = 2,      /* N the frame needs (may exceed the capacity it was given) */
  GAB200_CTR_NUM_LISTED = 3,        /* splats with at least one instance */
  GAB200_CTR_BUCKET_OVERFLOW = 4,   /* != 0: a depth bucket outgrew shared memory (depth_hint_* did not fit this frame) */
  GAB200_CTR_CAPACITY = 5,          /* capacity the binning stages ran with */
  GAB200_CTR_SEQ = 6,               /* caller's frame_seq echoed back: tells a finished copy from a stale one */
  GAB200_CTR_NUM_RENDERED_HI = 7,   /* bits 32.. of the instance total: non-zero = more than 2^32 - 1 instances (the 32-bit
                                       offsets wrapped: GAB200_ERR_OVERFLOW) */
  GAB200_NUM_COUNTERS = 8
};

typedef void* (*gab200_alloc_fn)(void* user, size_t bytes);

/* Everything one frame's forward needs.  Replaces the argument list of
 * diff_gaussian_rasterization._C.rasterize_gaussians (SURVEY.md 3.3 / Appendix B.6). */
typedef struct gab200_forward_args {
  uint32_t abi_version;    /* = GAB200_ABI_VERSION */
  int32_t input_mode;      /* gab200_input_mode */
  int32_t P;               /* number of splats */
  int32_t sh_degree;       /* active SH degree D (0..3) */
  int32_t sh_coeffs;       /* M: coefficients stored per splat (1,4,9,16); 0 with colors_precomp */
  int32_t image_width, image_height;
  float tanfovx, tanfovy;   /* tan(FoV / 2); the *_device_fov entry points read them from device memory instead */
  float scale_modifier;
  int32_t prefiltered;     /* accepted for signature parity; the near-plane cull is always applied */
  int32_t debug;           /* 1: synchronise + check after every stage (reference `debug=` flag) */
  int32_t need_backward;   /* 0: inference -- per-pixel state for backward is not written */
  int32_t binning_hint;    /* expected number of (splat,tile) instances (0 = unknown), e.g. last frame's N * 1.25.
                              GAB200_SYNC_EXACT: the binning buffer is requested BEFORE the host sync that reads N back
                              (allocation off the critical path; requested again only if N exceeds the hint).
                              GAB200_SYNC_LATE / NONE: the capacity the binning stages run with (see gab200_sync_mode) */
  int32_t exact_binning;   /* 1: emit the reference's full 3-sigma bounding-square instance list;
                              0: additionally drop (splat,tile) pairs that provably contribute nothing
                                 (alpha < 1/255 over the whole tile): image/gradients unchanged */
  uint32_t depth_hint_lo;  /* expected range of the visible splats' depth keys (fp32 bit patterns of view-space z), e.g.
                              the previous frame's gab200_frame_state.depth_key_min/max widened a little; hi <= lo = unknown.
                              With a hint the per-splat depth sort runs as a bucket sort (3 small launches) instead of
                              cub::DeviceRadixSort + DeviceScan (8 launches); the result is the same bit for bit, and a
                              hint that turns out wrong only costs the time of the radix path on top. */
  uint32_t depth_hint_hi;
  int32_t sync_mode;       /* gab200_sync_mode */
  uint32_t frame_seq;      /* any value; echoed in counters[GAB200_CTR_SEQ] */
  uint32_t* counters_host; /* HOST pointer (pinned memory), GAB200_NUM_COUNTERS words, or NULL: where the frame counters
                              are copied.  Required for GAB200_SYNC_NONE; the other modes fall back to a slot the
                              library keeps per host thread. */
  uint32_t* overflow_flag; /* DEVICE pointer or NULL: the library ORs 1 into it when the frame needed more than its
                              capacity or its depth buckets overflowed, and never clears it -- a replayed CUDA graph
                              (GAB200_SYNC_NONE) cannot lose an overflow between two looks at the counters */

  /* camera block */
  const float* bg;         /* [3] */
  const float* viewmatrix; /* [16] */
  const float* projmatrix; /* [16] */
  const float* campos;     /* [3] */

  /* splat attributes (meaning depends on input_mode) */
  const float* means3D;        /* [P,3]  world xyz | raw _xyz (face-local) */
  const float* opacities;      /* [P]    sigmoid-ed | raw logit */
  const float* scales;         /* [P,3]  exp-ed | raw log;            NULL iff cov3D_precomp */
  const float* rotations;      /* [P,4]  wxyz unit | raw unnormalised; NULL iff cov3D_precomp */
  const float* cov3D_precomp;  /* [P,6]  xx,xy,xz,yy,yz,zz; ACTIVATED mode only, else NULL */
  const float* shs;            /* [P,M,3] ACTIVATED mode: concatenated SH; NULL with colors_precomp */
  const float* sh_dc;          /* [P,1,3]   BOUND_RAW mode: _features_dc   (no torch.cat needed) */
  const float* sh_rest;        /* [P,M-1,3] BOUND_RAW mode: _features_rest (may be NULL when M==1) */
  const float* colors_precomp; /* [P,3]  overrides SH when non-NULL */

  /* mesh binding (BOUND_RAW mode; scene/flame_gaussian_model.py:137-147) */
  const int32_t* binding;        /* [P] face index per splat, or NULL (identity frame) */
  int32_t num_faces;             /* F */
  const float* face_center;      /* [F,3] */
  const float* face_orien_mat;   /* [F,3,3] row-major, columns a0 a1 a2 */
  const float* face_scaling;     /* [F] */

  /* outputs */
  float* out_color;   /* [3,H,W] */
  int32_t* radii;     /* [P] */
  uint8_t* visibility; /* [P] or NULL: radii > 0 as bytes -- render()'s `visibility_filter`
                          (gaussian_renderer/__init__.py:100) without a separate compare kernel */

  /* scratch (the reference's geomBuffer / binningBuffer / imgBuffer) */
  gab200_alloc_fn alloc_geom, alloc_binning, alloc_image;
  void* alloc_user;
} gab200_forward_args;

/* Host-side handle to the state a forward leaves behind for its backward (what the reference keeps as
 * num_rendered + the three byte buffers in the autograd ctx). Plain data; copy freely. */
typedef struct gab200_frame_state {
  int64_t num_rendered;       /* N: (splat,tile) instances sorted and blended */
  int64_t num_candidates;     /* instances of the reference's bounding-square list (== N when exact_binning) */
  void* geom_buffer;
  void* binning_buffer;
  void* image_buffer;
  size_t geom_bytes, binning_bytes, image_bytes;
  int32_t sorted_selector;    /* which half of the sort double-buffer holds the sorted stream */
  int32_t sort_bits;          /* key width of the per-instance (stage B) radix sort: bits(tile id) */
  int32_t depth_bits;         /* key width of the per-splat (stage A) radix sort: 32 (the fp32 depth pattern); the two
                                 stable stages together are the reference's LSD sort of (tile << 32 | depth) */
  uint32_t depth_prefix;      /* 1: a gab200_forward_depth_alpha or gab200_forward_views_train_depth_alpha frame kept for
                                 a backward -- its records carry the view-space depth that gab200_backward_depth_alpha /
                                 gab200_backward_views_depth_alpha read; 0 for every other forward */
  int64_t binning_capacity;   /* instances the binning buffer was carved for (>= num_rendered; = binning_hint when the
                                 speculative allocation was large enough) */
  uint32_t depth_key_min;     /* smallest / largest depth key among the splats that emitted instances (min > max: none) */
  uint32_t depth_key_max;
  int32_t depth_sort_path;    /* 0: radix sort (no hint); 1: bucket sort; 2: bucket sort overflowed, radix sort redone */
  int32_t attempts;           /* 1 + number of times stages were re-enqueued (GAB200_SYNC_LATE only; else 1) */
  int32_t tile_sort_path;     /* 0: cub::DeviceRadixSort over the instances; 1: counting sort by tile + per-tile rank sort */
  int32_t reserved0;          /* K of a gab200_forward_views_train frame (its backward is gab200_backward_views with the
                                 same K); 0 for every other forward */
  const uint32_t* device_counters; /* GAB200_NUM_COUNTERS words inside the geometry buffer (valid as long as it is) */
} gab200_frame_state;

/* Forward.  Returns num_rendered (>= 0) or a negative gab200_status.  With GAB200_SYNC_NONE the count is not known
 * when the call returns: it returns 0 and sets state_out->num_rendered = -1.  Enqueues on `stream` (cudaStream_t as
 * void*).  Host<->device synchronisation: see gab200_sync_mode. */
int64_t gab200_forward(const gab200_forward_args* args, gab200_frame_state* state_out, void* stream);

/* 1 if a GAB200_SYNC_NONE frame whose counters are in `counters` (HOST copy) was rendered from its complete instance
 * list, 0 if it overflowed (capacity or depth buckets) and has to be redone, -1 if the copy has not landed yet
 * (counters[GAB200_CTR_SEQ] != frame_seq). */
int32_t gab200_counters_ok(const uint32_t* counters, uint32_t frame_seq);

/* Gradients.  Replaces rasterize_gaussians_backward (SURVEY.md 3.4).  All outputs are written in full
 * (zeros where a splat received no gradient); NULL outputs are skipped where noted.
 * ACTIVATED mode: dL_dmeans3D [P,3], dL_dmeans2D [P,3] (x,y in NDC units, z = 0), dL_dopacity [P],
 *   dL_dcolors [P,3] (also the colors_precomp gradient), dL_dshs [P,M,3] | NULL, dL_dscales [P,3] | NULL,
 *   dL_drotations [P,4] | NULL, dL_dcov3D [P,6].
 * BOUND_RAW mode: same pointers are gradients w.r.t. the RAW parameters (_xyz, logit, log-scale, raw quaternion);
 *   dL_dsh_dc [P,1,3], dL_dsh_rest [P,M-1,3]; plus the face-frame gradients dL_dface_center [F,3],
 *   dL_dface_orien_mat [F,3,3], dL_dface_scaling [F] (accumulated; caller zero-initialises NOTHING -- the library does).
 */
typedef struct gab200_backward_args {
  uint32_t abi_version;
  const gab200_forward_args* fwd;   /* the same inputs the forward saw */
  const gab200_frame_state* state;
  const float* dL_dout_color;       /* [3,H,W] */
  float* dL_dmeans3D;
  float* dL_dmeans2D;
  float* dL_dopacity;
  float* dL_dcolors;
  float* dL_dshs;
  float* dL_dsh_dc;
  float* dL_dsh_rest;
  float* dL_dscales;
  float* dL_drotations;
  float* dL_dcov3D;
  float* dL_dface_center;
  float* dL_dface_orien_mat;
  float* dL_dface_scaling;
  /* Fused gradient all-reduce over NVLink/NVSwitch (BOUND_RAW mode, frame-sharded data parallel).  When 1, the six
   * parameter-gradient outputs (dL_dmeans3D, dL_drotations, dL_dscales, dL_dopacity, dL_dsh_dc, dL_dsh_rest) are
   * NVLS MULTICAST addresses of a symmetric buffer mapped on every rank of the group, and the kernel emits
   * multimem.red.add.f32 instead of stores: the switch sums the ranks' contributions while the backward kernel is
   * still running -- no separate all-reduce pass.  The caller zero-fills the buffer and barriers the group before
   * the call, and barriers again before reading the result (gaussianavatars_b200/dist.py does both).
   * Splats that received no gradient issue nothing (the buffer already holds their zero). */
  int32_t grads_are_multicast;
  /* Optional face-sorted view of `binding` (static between densifications, so the caller builds it once):
   * splats of one face are split into chunks (e.g. <= 16 splats); chunk c covers face_perm[face_chunk_start[c] ..
   * face_chunk_end[c]) and belongs to face face_chunk_face[c].  When given (num_face_chunks > 0), the face-frame
   * gradients are reduced per chunk by a second kernel instead of 13 global atomics per splat -- a face that owns
   * thousands of splats (hair, teeth) no longer serialises the L2 atomic unit. */
  const int32_t* face_perm;        /* [P] splat ids sorted by face */
  const int32_t* face_chunk_face;  /* [num_face_chunks] */
  const int32_t* face_chunk_start; /* [num_face_chunks] */
  const int32_t* face_chunk_end;   /* [num_face_chunks] */
  int32_t num_face_chunks;
} gab200_backward_args;

int32_t gab200_backward(const gab200_backward_args* args, void* stream);

/* Per-camera field of view read from device memory, so that one captured CUDA graph can render every camera of a
 * calibrated rig (the reference gives each camera its own FoVx / FoVy: scene/dataset_readers.py, render()).
 * tanfov: DEVICE float[2] = {tan(FoVx / 2), tan(FoVy / 2)}, 4-byte aligned, read by the kernels when they run -- a
 * graph replay uses whatever the caller wrote there before it.  args->tanfovx / tanfovy are ignored.  The arithmetic
 * after the load is that of gab200_forward: the same float values give bit-identical results.  A value that is zero,
 * negative or not finite culls every splat (radii 0, no instances, image = background); nothing is read or written
 * out of bounds.  tanfov == NULL: exactly gab200_forward / gab200_backward.  Every sync mode is supported.
 * The backward MUST be given the same pointer (holding the same values) as the forward whose state it consumes. */
int64_t gab200_forward_device_fov(const gab200_forward_args* args, const float* tanfov, gab200_frame_state* state_out,
                                  void* stream);
int32_t gab200_backward_device_fov(const gab200_backward_args* args, const float* tanfov, void* stream);

/* Forward whose blend also writes the display image: out_rgb8, a DEVICE uint8 [H,W,3] (row-major, RGB interleaved),
 * quantised as the reference's render.py does before it saves or shows a frame -- per channel of the float pixel c
 * (the value out_color receives), q = (uint8) clamp(c * 255 + 0.5, 0, 255) with the multiply and the add rounded
 * separately and truncation on the cast, i.e. torch's mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(uint8)
 * of out_color, bit for bit.  It is written by the forward blend itself: 3 bytes per pixel instead of 12, no extra
 * pass, and a D2H copy of the frame is a quarter of the float image's.
 * args->out_color may be NULL only when out_rgb8 is not NULL and args->need_backward == 0 (the float image is then
 * not written at all); any other NULL output is GAB200_ERR_INVALID_ARGUMENT.  tanfov: as gab200_forward_device_fov
 * (NULL: args->tanfovx / tanfovy).  out_rgb8 == NULL: exactly gab200_forward_device_fov.  Every sync mode is
 * supported; a frame the library re-enqueues (GAB200_SYNC_LATE) rewrites out_rgb8 with the EXACT frame's bytes. */
int64_t gab200_forward_display(const gab200_forward_args* args, const float* tanfov, uint8_t* out_rgb8,
                               gab200_frame_state* state_out, void* stream);

/* Opacity and depth beside the colour, from the same blend.  For each pixel the splats are walked exactly as the colour
 * blend walks them: the same list, the same alpha, the same 1/255 skip, the same T < 1e-4 stop.
 *   alpha = 1.0f - T_final, rounded once in fp32, where T_final is the transmittance the colour image uses as its
 *           background weight, so image = C + (1 - alpha) * bg holds exactly;
 *   depth = sum_i w_i z_i, accumulated as D = fmaf(z_i, w_i, D) in the same order and at the same point as the colour
 *           channels, with w_i = alpha_i T_i and z_i the splat's view-space depth (the fp32 value whose bits form its
 *           depth sort key: t.z = V[2] x + V[6] y + V[10] z + V[14] of the world-space mean).  Not normalised: a
 *           viewer's normalised depth is depth / alpha.  Inverse depth is not offered.
 * gab200_forward_depth_alpha is gab200_forward_display plus out_alpha and out_depth, DEVICE float [H,W] each; either may
 * be NULL, not both (GAB200_ERR_INVALID_ARGUMENT before any device work).  The colour image, display bytes, radii,
 * visibility and the backward state are those of gab200_forward_display bit for bit.  Every sync mode works; a frame
 * the library re-enqueues (GAB200_SYNC_LATE) rewrites both planes with the EXACT frame's values.  With need_backward,
 * state_out->depth_prefix = 1: the records carry z.
 * gab200_backward_depth_alpha is gab200_backward_device_fov (tanfov: the forward's, or NULL) plus dL_dalpha and
 * dL_ddepth, DEVICE float [H,W] each or NULL (= zero):
 *   dL/dalpha joins the background term: dL/dT_final gains -dL/dalpha;
 *   dL/ddepth is a fourth colour channel with c = z and bg = 0; each splat receives dL/dz = sum_pixels w dL/ddepth,
 *           which reaches the 3-D mean through t.z (then the binding chain and the face frame like every mean gradient);
 *   dL_dmeans2D includes the alpha and depth contributions (the gradient of the whole loss).
 * Before any device work, GAB200_ERR_INVALID_ARGUMENT for every error of gab200_backward, for a state whose
 * depth_prefix != 1 (a plain forward's, or a multi-view frame's) and for grads_are_multicast != 0.  gab200_backward on a
 * depth-alpha state is valid: the same backward with both plane gradients zero. */
int64_t gab200_forward_depth_alpha(const gab200_forward_args* args, const float* tanfov, float* out_alpha,
                                   float* out_depth, uint8_t* out_rgb8, gab200_frame_state* state_out, void* stream);
int32_t gab200_backward_depth_alpha(const gab200_backward_args* args, const float* tanfov, const float* dL_dalpha,
                                    const float* dL_ddepth, void* stream);

/* Every camera of a rig in one forward: `views` cameras render one splat set, the way a calibrated capture is
 * rendered and evaluated (all views of a timestep share the pose, so they need one pass, not one each).
 * cameras: DEVICE float[views][GAB200_CAMERA_FLOATS]; row k = world_view_transform (16) | full_proj_transform (16) |
 * camera_center (3) | tan(FoVx/2), tan(FoVy/2) -- the 37-float camera block with the field of view.  The kernels read
 * the table when they run, so a graph replay renders whatever was written there before it.  args->viewmatrix,
 * projmatrix, campos, tanfovx and tanfovy are ignored; image size, background, scale_modifier, SH degree and the splat
 * inputs (either input mode, colors_precomp included) are shared by all views.
 * Outputs: args->out_color [views,3,H,W] float and/or out_rgb8 [views,H,W,3] uint8 (quantised as gab200_forward_display
 * does); either may be NULL, not both.  args->radii [views,P]; args->visibility [views,P] or NULL.
 * The frame is K * P virtual splats -- splat i seen by camera k is virtual splat k * P + i and owns the global tiles
 * k * T .. k * T + T - 1 (T = tiles of one view) -- sorted and blended as one frame.  The stable per-splat depth sort
 * restricted to view k is camera k's own order and tiles of different views are disjoint, so every output (float
 * image, bytes, radii, visibility) is bit for bit that of `views` calls of gab200_forward_display with the same
 * cameras; views == 1 is that call.  A row whose tan(FoV/2) is zero, negative or not finite culls only its view (all
 * background).
 * Forward only: need_backward != 0 is GAB200_ERR_INVALID_ARGUMENT.  Every sync mode works as in gab200_forward;
 * binning_hint is the capacity of the whole K-view frame, and the counters, the sticky overflow_flag and the LATE
 * re-enqueue behave as documented there.  Before any device work, GAB200_ERR_INVALID_ARGUMENT for: views < 1 or
 * > 65535, cameras == NULL, views * P > INT32_MAX, views * T > INT32_MAX (the 32-bit tile key), and every error of
 * gab200_forward_display. */
#define GAB200_CAMERA_FLOATS 37
int64_t gab200_forward_views(const gab200_forward_args* args, int32_t views, const float* cameras, uint8_t* out_rgb8,
                             gab200_frame_state* state_out, void* stream);

/* Training over every camera of one timestep: the K-view frame of gab200_forward_views, kept for a backward.
 * It is gab200_forward_views with need_backward = 1 (args->need_backward is not read): args->out_color [views,3,H,W] is
 * required and no display image is written; radii [views,P] and visibility [views,P] | NULL as there.  Images, radii
 * and visibility are bit for bit those of gab200_forward_views and of `views` single-camera forwards.  The state keeps
 * what the backward reads for all K * P virtual splats and K * H * W pixels (final transmittance, contributor counts,
 * per-instance block masks, colour clamp bits, records) and records K in state_out->reserved0; the struct layout and
 * GAB200_ABI_VERSION are unchanged.  Every sync mode, binning_hint, the counters, the sticky overflow_flag and the
 * LATE re-enqueue behave as in gab200_forward_views.  Before any device work, GAB200_ERR_INVALID_ARGUMENT for every
 * error of gab200_forward_views except a NULL out_rgb8 (there is none), and for input_mode GAB200_INPUT_ACTIVATED and
 * colors_precomp != NULL: training uses BOUND_RAW splats with SH colours only. */
int64_t gab200_forward_views_train(const gab200_forward_args* args, int32_t views, const float* cameras,
                                   gab200_frame_state* state_out, void* stream);

/* Gradients of a gab200_forward_views_train frame, summed over its views: every output is what the sum over k of
 * gab200_backward of camera k's single-view frame would hold (float sums in another order).  args->fwd is the forward's
 * args, args->state its state, `views` and `cameras` the forward's (the table must hold the same values).
 * dL_dout_color [views,3,H,W]; dL_dmeans2D [views,P,3] | NULL (row k: camera k's dL/dmean2D, x,y in NDC units, z = 0);
 * dL_dmeans3D, dL_drotations, dL_dscales, dL_dopacity, dL_dsh_dc, dL_dsh_rest: the RAW-parameter gradients [P,...],
 * written in full (zeros where no view gave a gradient), each stored once -- one thread per splat sums the views in
 * order, without atomics.  dL_dface_* are zeroed and accumulated as in gab200_backward, through the CSR chunks when
 * given, else with atomics.  dL_dcolors, dL_dshs and dL_dcov3D are not read.
 * Before any device work, GAB200_ERR_INVALID_ARGUMENT for: views outside [1, 65535], cameras == NULL, every limit of
 * gab200_forward_views_train, a state whose reserved0 != views (a single-view state, or another K),
 * GAB200_INPUT_ACTIVATED, colors_precomp != NULL, grads_are_multicast != 0, a NULL dL_dout_color / dL_dsh_dc /
 * dL_dsh_rest (sh_coeffs > 1), and scratch buffers that are not the forward's.  gab200_backward and
 * gab200_backward_device_fov refuse a multi-view state. */
int32_t gab200_backward_views(const gab200_backward_args* args, int32_t views, const float* cameras, void* stream);

/* Opacity and depth for every camera of a K-view frame: the planes of gab200_forward_depth_alpha (same definitions, same
 * walk) for each view of gab200_forward_views / gab200_forward_views_train, and their gradients.
 * gab200_forward_views_depth_alpha is gab200_forward_views plus out_alpha and out_depth, DEVICE float [views,H,W] each
 * (view k's plane at offset k * H * W); either may be NULL, not both.  Every output is bit for bit that of `views` calls
 * of gab200_forward_depth_alpha with the same cameras (planes included), and colour, bytes, radii and visibility are
 * those of gab200_forward_views.  Before any device work, GAB200_ERR_INVALID_ARGUMENT for every error of
 * gab200_forward_views and for both planes NULL.
 * gab200_forward_views_train_depth_alpha is gab200_forward_views_train plus the two planes, as above.  The state records
 * K in state_out->reserved0 and sets state_out->depth_prefix = 1 (the records carry z).  Before any device work,
 * GAB200_ERR_INVALID_ARGUMENT for every error of gab200_forward_views_train and for both planes NULL.
 * Both forwards: every sync mode, binning_hint, the counters, the sticky overflow_flag and the LATE re-enqueue (which
 * rewrites both planes with the EXACT frame's values) behave as in gab200_forward_views.
 * gab200_backward_views_depth_alpha is gab200_backward_views plus dL_dalpha and dL_ddepth, DEVICE float [views,H,W]
 * each or NULL (= zero).  Every output is what the sum over k of gab200_backward_depth_alpha of camera k's single-view
 * frame would hold (float sums in another order): each view's dL/dz reaches the mean through that view's own view
 * matrix before the sums over the views.  Before any device work, GAB200_ERR_INVALID_ARGUMENT for every error of
 * gab200_backward_views and for a state whose depth_prefix != 1 (a plain K-view frame's).  gab200_backward_views on a
 * K-view depth-alpha state is valid: the colour backward, both plane gradients zero.  gab200_backward_depth_alpha
 * refuses a K-view state. */
int64_t gab200_forward_views_depth_alpha(const gab200_forward_args* args, int32_t views, const float* cameras,
                                         float* out_alpha, float* out_depth, uint8_t* out_rgb8,
                                         gab200_frame_state* state_out, void* stream);
int64_t gab200_forward_views_train_depth_alpha(const gab200_forward_args* args, int32_t views, const float* cameras,
                                               float* out_alpha, float* out_depth, gab200_frame_state* state_out,
                                               void* stream);
int32_t gab200_backward_views_depth_alpha(const gab200_backward_args* args, int32_t views, const float* cameras,
                                          const float* dL_dalpha, const float* dL_ddepth, void* stream);

/* Frustum test only.  Replaces diff_gaussian_rasterization._C.mark_visible (GaussianRasterizer.markVisible). */
int32_t gab200_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                            uint8_t* present /* [P] 0/1 */, void* stream);

/* Runs ONLY the binding + activation part of the fused preprocess (scene/gaussian_model.py:113-160) and exports
 * world-space means3D [P,3], opacities [P], scales [P,3] (exp * face scale) and cov3D [P,6] (with scale_modifier).
 * Any output may be NULL.  Same device code as the fused forward -> bit-identical values (parity tests, and the
 * callers that still need pc.get_xyz, e.g. convert_SHs_python). */
int32_t gab200_bind_activate(const gab200_forward_args* args, float* means3D, float* opacities, float* scales,
                             float* cov3D, void* stream);

/* Per-face frame of the posed mesh in one launch.  Replaces FlameGaussianModel.update_mesh_properties +
 * compute_face_orientation (scene/flame_gaussian_model.py:137-147, utils/graphics_utils.py:116-135):
 * verts [V,3], faces [F,3] int32 -> face_center [F,3], face_orien_mat [F,3,3] (columns a0 a1 a2), face_scaling [F]. */
int32_t gab200_face_frame_forward(int32_t F, int32_t V, const float* verts, const int32_t* faces, float* face_center,
                                  float* face_orien_mat, float* face_scaling, void* stream);
/* Its backward: dL/dverts [V,3] (zeroed by the library, then accumulated).  Any upstream gradient may be NULL (= 0). */
int32_t gab200_face_frame_backward(int32_t F, int32_t V, const float* verts, const int32_t* faces,
                                   const float* dL_dface_center, const float* dL_dface_orien_mat,
                                   const float* dL_dface_scaling, float* dL_dverts, void* stream);

/* Mean absolute error between a rendered image (n = 3*H*W floats) and a uint8 ground truth (value/255), with its
 * gradient, in one pass: *loss = mean |img - gt/255|, grad[i] = sign(img[i] - gt[i]/255) / n.  `loss` is zeroed by the
 * library.  Replaces `l1_loss(image, gt_image)` + its autograd and the float32 upload of the ground truth
 * (utils/loss_utils.py:17-18, train.py:128-131).  grad may be NULL (loss only). */
int32_t gab200_l1_loss_u8(int64_t n, const float* img, const uint8_t* gt, float* grad, float* loss, void* stream);
/* The gradient alone, scaled by an upstream gradient read from device memory (NULL = 1): grad[i] = *upstream *
 * sign(img[i] - gt[i]/255) / n.  What autograd's backward of the loss calls (grad may be NULL in the forward above:
 * loss only), so that no separate multiply pass runs over the (3,H,W) gradient. */
int32_t gab200_l1_loss_u8_backward(int64_t n, const float* img, const uint8_t* gt, const float* upstream, float* grad,
                                   void* stream);

/* The ground truth the reference's loader makes from a capture's RGBA frame (CameraDataset.__getitem__,
 * scene/__init__.py:48-51), in one launch: for every colour byte c and alpha byte a of `views` interleaved
 * [height, width, 4] uint8 frames,
 *   rgb_out = trunc((c / 255.0 * (a / 255.0) + bg[ch] * (1 - a / 255.0)) * 255.0)
 * evaluated in double precision in exactly that order (no contraction), written planar as [views, 3, height, width]
 * uint8 -- the loader's bytes, bit for bit -- and mask_out = a as [views, 1, height, width] uint8 (may be NULL).
 * bg: 3 floats in device memory, read on every launch.  The loader's backgrounds are 0 or 1 per channel; any other
 * colour goes through the same formula (converted to double), which the loader would give for that colour as well. */
int32_t gab200_composite_rgba(int64_t views, int32_t height, int32_t width, const uint8_t* rgba, const float* bg,
                              uint8_t* rgb_out, uint8_t* mask_out, void* stream);

/* The tile-packed lossless frame store (csrc/frames.cu, gaussianavatars_b200.frames.FrameStore): a frame is four
 * uint8 planes -- R, G, B of the composited ground truth, M its alpha (255 without a mask) -- coded per 16x16 tile
 * (row-major, edge-replicated) and plane as base = v(0,0), the mod-256 2-D difference d(y,x) = q(y,x) - q(y,x-1) -
 * q(y-1,x) + q(y-1,x-1) of q = v - base, zigzagged into b bits (b = bit length of the tile's largest residual).
 * Record, 8-byte aligned: 4 bases | uint16 of the 4 widths (plane p in bits 4p..4p+3) | 2 zero bytes | R, G, B, M
 * payloads of 32 b bytes (value 16 y + x at bits [i b, i b + b) of a little-endian bit stream): 8 + 32 sum(b) bytes.
 * Index: frame_base[f] (int64, byte offset into the arena), tile_off[f * n_tiles + t] (uint32, 8-byte units from the
 * frame's base).  n_tiles = ceil(height/16) * ceil(width/16).
 *
 * Plan: the record size, in 8-byte units, of every tile of `frames` frames gt [frames, 3, height, width] and mask
 * [frames, 1, height, width] (NULL: 255) -> record_units[frames * n_tiles]. */
int32_t gab200_frame_encode_plan(int64_t frames, int32_t height, int32_t width, const uint8_t* gt, const uint8_t* mask,
                                 uint32_t* record_units, void* stream);
/* Encode: the same frames' records, tile t of frame f at arena + frame_base[f] + 8 * tile_off[f * n_tiles + t] (the
 * caller's scan of the planned sizes; frame_base / tile_off here are the rows of the frames being encoded). */
int32_t gab200_frame_encode(int64_t frames, int32_t height, int32_t width, const uint8_t* gt, const uint8_t* mask,
                            const int64_t* frame_base, const uint32_t* tile_off, uint8_t* arena, void* stream);
/* Decode frames ids[0 .. views) (a device int32 table) -> gt_out [views, 3, height, width] and mask_out [views, 1,
 * height, width] (NULL: not written).  Reads nothing on the host: capturable.  The ids are not checked on the device:
 * each must index a frame of the arena. */
int32_t gab200_frame_decode(int32_t views, int32_t height, int32_t width, const int32_t* ids, const uint8_t* arena,
                            const int64_t* frame_base, const uint32_t* tile_off, uint8_t* gt_out, uint8_t* mask_out,
                            void* stream);

/* A device-resident view schedule (csrc/schedule.cu, gaussianavatars_b200.schedule.ViewSchedule): `records` records
 * of `views` cameras each -- cams [records, views, GAB200_CAMERA_FLOATS] float32, timesteps [records] int32 (may be
 * NULL), frame_ids [records, views] int32 (may be NULL) -- visited in the order order[0 .. length).  `cursor` is one
 * device int32, the iteration the next replay runs.  Both launches read nothing on the host: capturable.
 *
 * Sample (one CTA, a plain launch): c = *cursor, r = order[c]; cam_out [views, GAB200_CAMERA_FLOATS] = cams[r],
 * *timestep_out = timesteps[r], ids_out[k] = frame_ids[r * views + k], rows_out[k] = r * views + k (each output may
 * be NULL: not written; timestep_out / ids_out need their table).  If c lies outside [0, length) or r outside
 * [0, records), nothing is read or written but *exhausted = 1. */
int32_t gab200_schedule_sample(int32_t records, int32_t views, int32_t length, const float* cams,
                               const int32_t* timesteps, const int32_t* frame_ids, const int32_t* order,
                               const int32_t* cursor, float* cam_out, int32_t* timestep_out, int32_t* ids_out,
                               int32_t* rows_out, int32_t* exhausted, void* stream);
/* Commit (one thread, a plain launch at the end of the replay): nothing if *overflow_flag (may be NULL) or *exhausted
 * is set or *cursor lies outside [0, length); else losses[*cursor] = *loss (losses may be NULL: no log) and
 * *cursor += 1. */
int32_t gab200_schedule_commit(int32_t length, const int32_t* overflow_flag, const int32_t* exhausted,
                               const float* loss, float* losses, int32_t* cursor, void* stream);

/* Photometric training loss of the reference with its gradient, in two launches (SURVEY.md 8f rank 2):
 *   total = (1 - lambda_dssim) * mean|img - gt| + lambda_dssim * (1 - mean SSIM(img, gt))
 * Replaces `l1_loss(image, gt) * (1 - lambda)` + `(1 - ssim(image, gt)) * lambda` and their autograd
 * (utils/loss_utils.py:17-18,36-63; train.py:131-132): 11x11 Gaussian window, sigma 1.5, zero padding, C1 = 0.01^2,
 * C2 = 0.03^2, mean over all channels and pixels.  image / grad: float32 [channels, height, width]; gt: the same
 * shape as uint8 (value/255; gt_is_u8 = 1) or float32 (gt_is_u8 = 0).  loss[3] receives {L1 mean, SSIM mean, total}
 * scratch: GAB_PHOTOMETRIC_SCRATCH_HEAD + 3 * channels * height * width floats owned by the caller, 16-byte aligned
 * (two double accumulators, then the three partial-derivative maps handed from the first launch to the second). */
#define GAB_PHOTOMETRIC_SCRATCH_HEAD 4
typedef struct gab200_photometric_args {
  uint32_t abi_version;
  int32_t channels, height, width;
  int32_t gt_is_u8;
  float lambda_dssim;
  const float* image;
  const void* gt;
  float* grad;    /* [channels, height, width]  d total / d image */
  float* loss;    /* [3] */
  float* scratch; /* [GAB_PHOTOMETRIC_SCRATCH_HEAD + 3 * channels * height * width] */
} gab200_photometric_args;
int32_t gab200_photometric_loss(const gab200_photometric_args* args, void* stream);

/* Image metrics of one rendered view against its ground truth, forward only, in two launches with no host wait.
 * Replaces the evaluation the reference runs per val / test view in training_report (train.py:277-288: clamp(0, 1) of
 * the render, then l1_loss, psnr and ssim) and in metrics.py:71-74 (ssim and psnr of the PNG render.py wrote, read
 * back as value/255): utils/image_utils.py:18-20 and utils/loss_utils.py:33-63 (11x11 Gaussian window, sigma 1.5,
 * zero padding, C1 = 0.01^2, C2 = 0.03^2 -- the arithmetic of gab200_photometric_loss's SSIM).
 *   render_kind GAB200_METRICS_FLOAT_CHW: render is float32 [3,H,W], clamped to [0, 1] in-kernel (train.py:277).
 *   render_kind GAB200_METRICS_U8_HWC:    render is the display image uint8 [H,W,3] (gab200_forward_display), read as
 *                                         value/255 correctly rounded (render.py's PNG bytes through to_tensor).
 *   gt: uint8 [3,H,W], value/255 (PILtoTorch).
 * The record written is GAB200_METRICS_FIELDS floats:
 *   [0] l1       mean |render - gt| over all 3HW values
 *   [1] psnr     mean over the three channels of 20 log10(1 / sqrt(MSE of the channel)): train.py passes a [3,H,W]
 *                image to psnr(), whose view(img1.shape[0], -1) makes one PSNR per channel, then .mean()
 *   [2] psnr_all 20 log10(1 / sqrt(MSE over all 3HW values)): metrics.py passes [1,3,H,W] tensors
 *   [3] ssim     mean of the SSIM map over all 3HW values
 * An MSE of 0 gives +inf.  Sums run in double and are reduced in a fixed order (no floating-point atomics): the same
 * inputs give bit-identical records on every call.
 * The record goes to row *row of `table` ([table_rows, GAB200_METRICS_FIELDS] float32); row is a DEVICE int32 read
 * when the kernel runs (NULL = row 0), so a replayed CUDA graph can write a different row each time.  A row outside
 * [0, table_rows) writes nothing.  skip_flag: DEVICE pointer or NULL, as gab200_adam_step_device: non-zero when the
 * kernel runs = nothing is written (a graph replay whose render overflowed its instance capacity leaves its row as it
 * was).  scratch: gab200_image_metrics_scratch_bytes(height, width) bytes of device memory, 8-byte aligned.
 * Invalid arguments (GAB200_ERR_INVALID_ARGUMENT): a NULL args, render, gt, table or scratch, a non-positive height
 * or width, table_rows < 1, an unknown render_kind, abi_version != GAB200_ABI_VERSION. */
#define GAB200_METRICS_FIELDS 4
typedef enum gab200_metrics_render_kind {
  GAB200_METRICS_FLOAT_CHW = 0,
  GAB200_METRICS_U8_HWC = 1
} gab200_metrics_render_kind;
typedef struct gab200_metrics_args {
  uint32_t abi_version;
  int32_t height, width;
  int32_t render_kind;      /* gab200_metrics_render_kind */
  const void* render;       /* float [3,H,W] | uint8 [H,W,3] */
  const uint8_t* gt;        /* [3,H,W] */
  const int32_t* row;       /* DEVICE int32 or NULL (= 0) */
  float* table;             /* [table_rows, GAB200_METRICS_FIELDS] */
  int32_t table_rows;
  const int32_t* skip_flag; /* DEVICE int32 or NULL */
  void* scratch;
} gab200_metrics_args;
size_t gab200_image_metrics_scratch_bytes(int32_t height, int32_t width);
int32_t gab200_image_metrics(const gab200_metrics_args* args, void* stream);

/* LPIPS distance (v0.1) of one rendered view against its ground truth, forward only, with no host wait (capturable).
 * Replaces lpipsPyTorch's LPIPS as the reference calls it: AlexNet in training_report (train.py:290-302, per val / test
 * view of the clamped render), VGG-16 in metrics.py:74 (the PNG bytes render.py wrote, read back as value/255).
 *   Input: render and gt as gab200_image_metrics reads them (render_kind, clamp, value/255), each z-scored as
 *     (x - (-.030, -.088, -.188)) / (.458, .448, .450) in float32 -- on [0, 1] inputs, as the reference does.
 *   Network: torchvision's alexnet().features / vgg16().features up to the last target ReLU; the targets are the
 *     ReLU before each pool and the last one (AlexNet relu1..relu5; VGG-16 relu1_2, relu2_2, relu3_3, relu4_3,
 *     relu5_3).  Convolutions run on the tensor cores with TF32 operands rounded to nearest and FP32 accumulation,
 *     the K loop in one fixed order; pools are exact.
 *   Head: per target pixel f / (sqrt(sum_c f^2) + 1e-10) of both images, the squared difference, the lin layer's
 *     dot product (FP32); per layer the mean over the pixels (sums in double, fixed order); the five means summed.
 * The distance goes to table[*row] ((table_rows,) float32; row is a DEVICE int32, NULL = 0; a row outside
 * [0, table_rows) writes nothing), unless *skip_flag (DEVICE int32 or NULL) is non-zero when the kernel runs.  No
 * floating-point atomics: the same inputs and weights give bit-identical results on every call.
 * weights: gab200_lpips_weights_bytes(net) bytes filled by gab200_lpips_pack, 16-byte aligned.
 * scratch: gab200_lpips_scratch_bytes(net, height, width) bytes, 16-byte aligned: the per-CTA partial sums and two
 *   activation buffers of both images (VGG-16 at 1920x1080: 2 x 1.06 GB).
 * features: NULL, or a 16-byte aligned buffer of gab200_lpips_features_bytes(net, height, width) bytes that receives
 *   every stage's output in float32, in order -- the
 *   z-scored input (4 channels, the 4th 0), then each convolution's post-ReLU output and each pool's output -- each as
 *   [2][H_s][W_s][C_s] (image 0 the render, image 1 the ground truth).  A test surface: the stages then write there
 *   instead of the scratch buffers.
 * gab200_lpips_scratch_bytes and gab200_lpips_features_bytes are 0 for an unknown net, and for an image the network
 * cannot take: below 31 x 31 (AlexNet) or 16 x 16 (VGG-16) in either side.
 * Invalid arguments (GAB200_ERR_INVALID_ARGUMENT): a NULL args, render, gt, weights, table or scratch, a misaligned
 * weights, scratch or features, an unknown net or render_kind, a size gab200_lpips_scratch_bytes refuses,
 * table_rows < 1, abi_version != GAB200_ABI_VERSION. */
typedef enum gab200_lpips_net {
  GAB200_LPIPS_ALEX = 0,
  GAB200_LPIPS_VGG16 = 1
} gab200_lpips_net;
typedef struct gab200_lpips_args {
  uint32_t abi_version;
  int32_t net;              /* gab200_lpips_net */
  int32_t height, width;
  int32_t render_kind;      /* gab200_metrics_render_kind */
  const void* render;       /* float [3,H,W] | uint8 [H,W,3] */
  const uint8_t* gt;        /* [3,H,W] */
  const void* weights;      /* gab200_lpips_pack's buffer */
  const int32_t* row;       /* DEVICE int32 or NULL (= 0) */
  float* table;             /* [table_rows] */
  int32_t table_rows;
  const int32_t* skip_flag; /* DEVICE int32 or NULL */
  void* scratch;
  float* features;          /* NULL, or every stage's output (see above) */
} gab200_lpips_args;
/* Bytes of the packed weights of a network (0 for an unknown net). */
size_t gab200_lpips_weights_bytes(int32_t net);
/* Packs a network's weights once: conv_weight[l] / conv_bias[l] are DEVICE pointers to torchvision's float32
 * features.N.weight (OIHW, contiguous) and features.N.bias of the l-th convolution up to the last target (5 for AlexNet,
 * 13 for VGG-16), lin_weight[t] the t-th lin layer's (C_t) float32 weights; the pointer arrays themselves are host
 * memory.  packed: gab200_lpips_weights_bytes(net) bytes, 16-byte aligned.  Stream-ordered, no host wait. */
int32_t gab200_lpips_pack(int32_t net, const float* const* conv_weight, const float* const* conv_bias,
                          const float* const* lin_weight, void* packed, void* stream);
size_t gab200_lpips_scratch_bytes(int32_t net, int32_t height, int32_t width);
size_t gab200_lpips_features_bytes(int32_t net, int32_t height, int32_t width);
int32_t gab200_lpips(const gab200_lpips_args* args, void* stream);

/* The tracked mesh drawn over an image, forward only, in four launches with no host wait (capturable).  Replaces
 * what the reference's mesh renderer (mesh_renderer/__init__.py:183-274) asks of nvdiffrast -- dr.rasterize and
 * dr.antialias -- and, fused, render.py's mesh composite (render.py:75-81) and its uint8 quantisation.
 *   Geometry.  pos_kind GAB200_MESH_POS_WORLD: verts [V,3] world space, clip = [v,1] . full_proj_transform (the 16
 *     floats at camera + 16; camera is the 35- or 37-float camera block world_view (16) | full_proj (16) | centre (3)
 *     [| tan fov (2)]).  GAB200_MESH_POS_CLIP: verts [V,4] are clip coordinates (nvdiffrast's `pos`); camera unused.
 *     Faces [F,3] int32.  A face is clipped against -w <= z <= w (nvdiffrast's clip volume) and a guard band of 2^15
 *     pixels, and its vertices are snapped to 1/256 pixel.  Coverage: int64 edge functions at pixel centres with a
 *     top-left fill rule -- watertight, no pixel covered twice along a shared edge.  No back-face culling.  Depth: z/w
 *     at the pixel centre; the nearest face wins, ties go to the smaller face index.
 *   Pixels.  Column c / row r has its centre at (c + 1/2, r + 1/2) with X = (x/w + 1) W / 2, Y = (y/w + 1) H / 2: row 0
 *     is clip y = -1 (the top row of the splat image for a camera's own full_proj_transform; nvdiffrast's row 0 for
 *     the reference's y-negated clip coordinates).  Images are row-major in that order.
 *   Shading (POS_WORLD).  n = normalize(cross(v1 - v0, v2 - v0)) in the OpenGL camera frame (rows 1, 2 of the view
 *     transform negated); diffuse = clamp(n.z, 0, 1) (GAB200_MESH_LIGHT_FRONT) or 1 (GAB200_MESH_LIGHT_CONSTANT);
 *     rgba = (face_colors[f] (or 1) * diffuse, 1) where covered, (background, 0) elsewhere.
 *   Antialiasing (antialias = 1; needs adjacency).  For every pair of horizontally or vertically adjacent pixels whose
 *     winners differ, the occluder is the pixel whose face is nearer at its own centre (a covered pixel occludes the
 *     background).  The occluder face's silhouette edges -- a mesh boundary, or the face across the edge lies on the
 *     same side of the edge's projected line; a face with a vertex outside the clip volume has none -- with
 *     |dx| <= |dy| are tested on horizontal pairs, the others on vertical ones: t = e(a) / (e(a) - e(b)), the crossing
 *     on the segment between the centres counted from the occluder a, must lie in [0, 1] and within the edge's extent;
 *     the smallest t wins.  t < 1/2: a moves toward b by 1/2 - t; t > 1/2: b moves toward a by t - 1/2.  Every delta is
 *     taken from the un-antialiased colours and a pixel adds its deltas in the order left, right, up, down (no atomics:
 *     the same inputs give the same bits).  This is the silhouette-coverage approximation of Laine et al. 2020,
 *     "Modular Primitives for High-Performance Differentiable Rendering", section 3.3; it is not claimed to equal
 *     nvdiffrast bit for bit.
 *   adjacency [F,3] int32: adjacency[f][k] = the face across edge k = (faces[f][k], faces[f][(k+1) % 3]), or -1 when
 *     no face or more than one other face shares that edge (a boundary).  It depends on faces only: build it once.
 * Outputs (any may be NULL; at least one is required):
 *   out_rgba  [H,W,4] float: the antialiased rgba (the reference's `rgba` before its flip)     POS_WORLD
 *   out_u8    [H,W,3] uint8 / out_float [3,H,W] float: the composite
 *               rgb * a * o + base * (a * (1 - o) + (1 - a))
 *             in torch's evaluation order, every op rounded (render.py's expression), out_u8 quantised as render.py
 *             does (mul(255).add_(0.5).clamp_(0, 255), truncation).  base: float [3,H,W] (GAB200_MESH_BASE_FLOAT_CHW)
 *             or uint8 [3,H,W] read as value/255 correctly rounded (GAB200_MESH_BASE_U8_CHW).  opacity: DEVICE
 *             float[2] = {o, 1 - o}, both rounded from the caller's double, as torch rounds its Python scalars;
 *             read when the kernel runs (a replayed graph picks up a new opacity)                  POS_WORLD
 *   out_rast  [H,W,4] float: nvdiffrast's rast_out -- perspective-correct barycentrics (u, v) of the original
 *             triangle's vertices 0 and 1, z/w, face index + 1; zeros where nothing is covered
 *   out_color [H,W,channels] float: antialias of the caller's image in_color [H,W,channels] (1..64 channels)
 * in_rast [H,W,4] or NULL: the winners are taken from this rast_out (channel 2 z/w, channel 3 face index + 1) instead of
 *   being rasterized: nvdiffrast's antialias(color, rast, pos, tri).
 * error_flag: DEVICE int32 or NULL: 1 is ORed into it when a face has a vertex index outside [0, V); that face is not
 *   drawn and nothing is read out of bounds.
 * scratch: gab200_mesh_scratch_bytes(F, width, height) bytes of device memory, 256-byte aligned.
 * Invalid arguments (GAB200_ERR_INVALID_ARGUMENT): abi_version, V < 1, F < 1, width / height outside [1, 16384], a
 * NULL verts / faces / scratch, an unknown pos_kind / lighting / base_kind, POS_WORLD without camera, antialias
 * without adjacency, no output, out_rgba / out_u8 / out_float with POS_CLIP, out_u8 / out_float without base or
 * opacity, out_color without in_color or a channel count outside [1, 64]. */
typedef enum gab200_mesh_pos_kind { GAB200_MESH_POS_WORLD = 0, GAB200_MESH_POS_CLIP = 1 } gab200_mesh_pos_kind;
typedef enum gab200_mesh_lighting { GAB200_MESH_LIGHT_FRONT = 0, GAB200_MESH_LIGHT_CONSTANT = 1 } gab200_mesh_lighting;
typedef enum gab200_mesh_base_kind {
  GAB200_MESH_BASE_NONE = 0,
  GAB200_MESH_BASE_FLOAT_CHW = 1,
  GAB200_MESH_BASE_U8_CHW = 2
} gab200_mesh_base_kind;
typedef struct gab200_mesh_args {
  uint32_t abi_version;
  int32_t V, F, width, height;
  int32_t pos_kind;            /* gab200_mesh_pos_kind */
  const float* verts;          /* [V,3] | [V,4] */
  const int32_t* faces;        /* [F,3] */
  const int32_t* adjacency;    /* [F,3] or NULL (antialias = 0) */
  const float* camera;         /* camera block (POS_WORLD) */
  const float* face_colors;    /* [F,3] or NULL (albedo 1) */
  float background[3];
  int32_t lighting;            /* gab200_mesh_lighting */
  int32_t antialias;           /* 0 | 1 */
  int32_t base_kind;           /* gab200_mesh_base_kind */
  const void* base;
  const float* opacity;        /* DEVICE float[2] = {o, 1 - o} */
  uint8_t* out_u8;             /* [H,W,3] */
  float* out_float;            /* [3,H,W] */
  float* out_rgba;             /* [H,W,4] */
  float* out_rast;             /* [H,W,4] */
  const float* in_rast;        /* [H,W,4] or NULL */
  const float* in_color;       /* [H,W,channels] or NULL */
  float* out_color;            /* [H,W,channels] */
  int32_t channels;
  int32_t* error_flag;         /* DEVICE int32 or NULL */
  void* scratch;
} gab200_mesh_args;
size_t gab200_mesh_scratch_bytes(int32_t num_faces, int32_t width, int32_t height);
int32_t gab200_mesh_render(const gab200_mesh_args* args, void* stream);

/* Adam over several parameter arrays in one launch (SURVEY.md 8f rank 3).  Replaces `gaussians.optimizer.step()` for
 * the splat parameter groups (scene/gaussian_model.py:213-232 builds `torch.optim.Adam(l, lr=0.0, eps=1e-15)` with one
 * group -- and one learning rate -- per array; train.py:207-209): amsgrad off, no weight decay, bias-corrected, `step`
 * counts from 1.  `segments` is a HOST array; every pointer inside is a device pointer to n floats. */
#define GAB_ADAM_MAX_SEGMENTS 8 /* per launch; longer lists are split */
typedef struct gab200_adam_segment {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t n;
  double lr; /* hyper-parameters travel as double, like the Python floats torch forms its scalars from */
} gab200_adam_segment;
int32_t gab200_adam_step(int32_t num_segments, const gab200_adam_segment* segments, int64_t step, double beta1,
                         double beta2, double eps, void* stream);

/* The same Adam step with nothing read from the host per step, so that it can be captured into a CUDA graph and
 * replayed (torch's `capturable=True` layout).  Every segment owns a device float32 step counter (distinct per
 * segment); the call first increments every counter on the device (one single-thread launch), then the Adam launch
 * forms bias_correction1/2 and lr / bias_correction1 in double from the segment's new step -- the arithmetic of
 * gab200_adam_step -- and rounds them to float once.  A segment with has_schedule = 1 takes its learning rate from
 * the reference's exponential schedule (utils/general_utils.py get_expon_lr_func, evaluated in double at the new step:
 * in train.py the optimizer steps once per iteration from 1, so that step is the iteration); otherwise from `lr`.
 * skip_flag: DEVICE pointer or NULL.  When non-NULL and *skip_flag != 0 at execution time, both launches write
 * nothing (no parameter, moment or step changes): a graph replay whose render overflowed its instance capacity
 * (gab200_forward_args.overflow_flag) leaves the model untouched instead of applying wrong gradients.  Empty segments
 * (n = 0) still count a step, as torch does. */
typedef struct gab200_adam_device_segment {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t n;
  float* step;            /* device float32 scalar */
  double lr;              /* constant learning rate (has_schedule = 0) */
  int32_t has_schedule;
  int32_t reserved0;
  double lr_init, lr_final, lr_delay_mult;   /* get_expon_lr_func(lr_init, lr_final, lr_delay_steps, lr_delay_mult, */
  int64_t lr_delay_steps, max_steps;         /*                   max_steps); max_steps > 0                          */
} gab200_adam_device_segment;
int32_t gab200_adam_step_device(int32_t num_segments, const gab200_adam_device_segment* segments, double beta1,
                                double beta2, double eps, const int32_t* skip_flag, void* stream);

/* The position / scale regularisers of the mesh-bound training step (train.py:134-146), loss and gradient in one
 * launch each.  vis = radii > 0 of the frame just rendered.  loss[3] receives {xyz term, scale term, visible count};
 * sums: 3 doubles of device scratch shared by the forward and its backward.  The backward writes grad_xyz /
 * grad_scaling [P,3] in full (zeros for invisible splats) and ADDS into grad_face_scaling [F] (metric_* only; the
 * caller zero-fills it); g_out[2] = upstream gradients of the two terms (device). */
typedef struct gab200_regularize_args {
  uint32_t abi_version;
  int32_t P;
  int32_t metric_xyz, metric_scale;
  float threshold_xyz, threshold_scale, lambda_xyz, lambda_scale;
  const float *xyz, *scaling;          /* raw _xyz, _scaling [P,3] */
  const int32_t* radii;                /* [P] */
  const int32_t* binding;              /* [P] or NULL */
  const float* face_scaling;           /* [F] */
  float* loss;                         /* [3] */
  double* sums;                        /* [3] */
  float *grad_xyz, *grad_scaling, *grad_face_scaling;   /* backward only */
} gab200_regularize_args;
int32_t gab200_regularize_forward(const gab200_regularize_args* args, void* stream);
int32_t gab200_regularize_backward(const gab200_regularize_args* args, const float* g_out, void* stream);

/* In-place all-reduce (sum) of n floats that every rank of a group holds in NVLink symmetric memory, through the
 * NVSwitch multicast address `mc_ptr` of that allocation (NVLS): rank r reduces the r-th slice with
 * multimem.ld_reduce and stores it to every replica with multimem.st.  16-byte aligned.  The CALLER orders it between
 * two group barriers on the stream (every replica written before / every slice stored after): dist.py uses the
 * symmetric-memory signal pads.  Replaces the ncclAllReduce of the flat splat-gradient buffer (SURVEY.md 8e). */
int32_t gab200_nvls_allreduce(float* mc_ptr, int64_t n, int32_t rank, int32_t world, void* stream);

/* densify_and_prune of the splat arrays with the Adam-state surgery fused (SURVEY.md 8f rank 3).  Replaces
 * GaussianModel.densify_and_prune (scene/gaussian_model.py:503-519 -> densify_and_clone :481-501, densify_and_split
 * :451-479, prune_points :371-397) together with the optimizer surgery it drives (:334-369, :399-424) and the
 * binding / binding_counter bookkeeping (:375-380, :395-397, :472-474, :495-497).  Two calls, because the caller has to
 * size the outputs:
 *   gab200_densify_plan   classifies every splat and scans the result; performs ONE stream synchronisation and leaves
 *                         totals_host = {kept originals, kept clones, kept child pairs, split parents}.
 *                         Output rows: P' = totals[0] + totals[1] + 2 * totals[2], in the reference's order
 *                         (originals, clones, first children, second children).
 *   gab200_densify_apply  gathers the six parameter arrays and their exp_avg / exp_avg_sq into the outputs (new rows get
 *                         zero moments), samples the children (noise: [2 * totals[3], 3] STANDARD normal values, rows
 *                         [0, S) for the first child of the S split parents in index order, [S, 2S) for the second --
 *                         exactly what torch.normal(mean=0, std=...) draws), and rebuilds binding / binding_counter.
 * The densification statistics (xyz_gradient_accum, denom, max_radii2D) of the result are all zero in the reference
 * (densification_postfix :447-449): the caller allocates zeros of length P'. */
typedef struct gab200_densify_args {
  uint32_t abi_version;
  int32_t P, num_faces;
  int32_t sh_rest_width;   /* floats per splat of _features_rest: 3 * (M - 1) */
  float grad_threshold, min_opacity, extent, percent_dense;
  float max_screen_size;   /* <= 0: None */
  const float *xyz, *rotation, *scaling, *opacity, *f_dc, *f_rest;   /* raw parameters [P, 3|4|3|1|3|sh_rest_width] */
  const float* exp_avg[6];     /* Adam moments in the order xyz, rotation, scaling, opacity, f_dc, f_rest; NULL = none */
  const float* exp_avg_sq[6];
  const float *xyz_gradient_accum, *denom;   /* [P] */
  const int32_t* binding;          /* [P] or NULL (plain GaussianModel) */
  const int32_t* binding_counter;  /* [F] */
  const float* face_scaling;       /* [F] */
  void* scratch;                   /* device, gab200_densify_scratch_bytes(P, F) bytes, 256-byte aligned; shared by both calls */
  uint32_t* totals_host;           /* HOST (pinned), 4 words */
} gab200_densify_args;
typedef struct gab200_densify_out {
  int32_t P_out, n_child_rows;     /* totals[0] + totals[1] + 2 totals[2];  2 totals[2] */
  float *xyz, *rotation, *scaling, *opacity, *f_dc, *f_rest;
  float* exp_avg[6];
  float* exp_avg_sq[6];
  int32_t* binding;                /* [P_out] or NULL */
  int32_t* binding_counter;        /* [F] or NULL */
  const float* noise;              /* [2 * totals[3], 3] */
  int32_t* src_scratch;            /* [P_out] device scratch */
  uint8_t* kind_scratch;           /* [P_out] */
  int32_t* noise_row_scratch;      /* [totals[2]] */
} gab200_densify_out;
size_t gab200_densify_scratch_bytes(int32_t P, int32_t num_faces);

/* The densification statistics of one rendered frame, in place, in one launch over the P splats (no mask, no
 * compaction, no host wait).  For every splat with radii > 0:
 *   max_radii2D = max(max_radii2D, float(radii))                                   (train.py:197)
 *   xyz_gradient_accum += ||viewspace_grad[:, :2]||,  denom += 1                    (scene/gaussian_model.py:517-519)
 * viewspace_grad [P,3] (viewspace_points.grad), radii [P] int32, xyz_gradient_accum [P,1], denom [P,1],
 * max_radii2D [P].  skip_flag: as gab200_adam_step_device (DEVICE pointer or NULL; non-zero = write nothing). */
int32_t gab200_densify_stats(int32_t P, const float* viewspace_grad, const int32_t* radii, float* xyz_gradient_accum,
                             float* denom, float* max_radii2D, const int32_t* skip_flag, void* stream);
int32_t gab200_densify_plan(const gab200_densify_args* args, void* stream);
int32_t gab200_densify_apply(const gab200_densify_args* args, const gab200_densify_out* out, void* stream);

/* FLAME head posing: blendshapes and linear blend skinning, forward and backward, for one timestep read from device
 * memory.  Replaces FlameHead.forward + lbs (flame_model/flame.py:485-558, flame_model/lbs.py:25-304) as
 * select_mesh_by_timestep calls it (scene/flame_gaussian_model.py:117-135): zero_centered_at_root_node = False,
 * no landmarks, translation added after skinning, full_pose = [rotation, neck, jaw, eyes (6)],
 * pose feature = (R_1..R_4 - I) flattened row-major, Rodrigues as lbs.py writes it (angle = |r + 1e-8|, exactly I at
 * r = 0 with a finite gradient).  The reference's dynamic_offset argument is accepted there and never used, so it has
 * no counterpart here.
 *
 * Only FLAME's kinematic layout is accepted: J = 5 joints (root, neck, jaw, two eyes), parents[0] = -1,
 * 0 <= parents[i] < i, 36 = 9 (J - 1) pose-basis rows; 0 <= n_shape, 0 <= n_expr <= GAB200_FLAME_MAX_EXPR.
 * Anything else is GAB200_ERR_INVALID_ARGUMENT.  All device arrays are float32 in the reference FlameHead buffer
 * layouts:
 *   v_template [V,3], shapedirs [V,3,n_shape+n_expr], posedirs [36,3V] (flame.py:117-119), J_regressor [J,V],
 *   lbs_weights [V,J]. */
#define GAB200_FLAME_J 5
#define GAB200_FLAME_POSE_BASIS 36
#define GAB200_FLAME_MAX_EXPR 100
#define GAB200_FLAME_FRAME_FLOATS 128 /* per-call state: A [5,3,4] | pose feature [36] | posed joints [5,3] | pad */
typedef struct gab200_flame_assets {
  uint32_t abi_version;
  int32_t V, n_shape, n_expr, J;
  int32_t parents[GAB200_FLAME_J]; /* HOST ints */
  const float* v_template;
  const float* shapedirs;
  const float* posedirs;
  const float* J_regressor;
  const float* lbs_weights;
} gab200_flame_assets;

/* Device scratch owned by the caller (256-byte aligned) holding what gab200_flame_prepare derives from the shape
 * and the static offset, plus the backward's per-CTA partial sums.  One scratch serves one stream at a time. */
size_t gab200_flame_scratch_bytes(int32_t V, int32_t n_expr);

/* Run once per change of `shape` [n_shape] or `static_offset` [V,3] (NULL = zero), which the reference never trains
 * (their optimizer groups are commented out, scene/flame_gaussian_model.py:180-183,209-217).  Writes into scratch:
 *   v_base = v_template + shapedirs[..., :n_shape] . shape + static_offset     [V,3]
 *   J_base = J_regressor . v_base                                              [5,3]
 *   JS     = J_regressor . shapedirs[..., n_shape:]                            [5,3,n_expr]
 *   the expression basis re-laid out component-major [n_expr,3V] for coalesced per-frame reads.
 * This regroups the reference's sums (one einsum over all n_shape + n_expr components, then the joints regressed from
 * the float32 v_shaped): results agree with it to rounding, not bit for bit. */
int32_t gab200_flame_prepare(const gab200_flame_assets* assets, const float* shape, const float* static_offset,
                             void* scratch, void* stream);

/* One timestep of the reference's flame_param dict: the (T,.) tensors and the row index t in DEVICE memory, so that
 * a captured CUDA graph poses whichever timestep the caller wrote before the replay.  A t outside [0, T) leaves the
 * outputs unspecified but is memory-safe: every kernel returns without reading a parameter row or writing. */
typedef struct gab200_flame_frame_args {
  uint32_t abi_version;
  int32_t T;
  const gab200_flame_assets* assets;
  const void* scratch;        /* prepared by gab200_flame_prepare for this shape / static offset */
  const int32_t* timestep;    /* DEVICE int32 */
  const float* expr;          /* [T, n_expr] */
  const float* rotation;      /* [T, 3] */
  const float* neck_pose;     /* [T, 3] */
  const float* jaw_pose;      /* [T, 3] */
  const float* eyes_pose;     /* [T, 6] */
  const float* translation;   /* [T, 3] */
  float* frame;               /* [GAB200_FLAME_FRAME_FLOATS] device: written by the forward, read by its backward */
} gab200_flame_frame_args;

/* Two launches, no host read: flame_joints_kernel (one CTA: joints, Rodrigues, rigid chain, pose feature) and
 * flame_skin_kernel (blendshapes, pose correctives, skinning).  verts [V,3]; verts_cano [V,3] (the reference's
 * v_shaped, returned for the laplacian term) or NULL. */
int32_t gab200_flame_forward(const gab200_flame_frame_args* args, float* verts, float* verts_cano, void* stream);

/* Gradients of the six (T,.) tensors, written in FULL: row t, and exact zeros in every other row (what autograd of the
 * reference's [[timestep]] indexing produces).  dL_dverts [V,3]; dL_dverts_cano [V,3] or NULL (= 0).  Two launches
 * (flame_skin_backward_kernel: per-CTA partial sums; flame_joints_backward_kernel: one CTA sums them in a fixed order
 * and backpropagates through the chain and Rodrigues), no floating-point atomics: the same dL_dverts gives
 * bit-identical gradients on every call. */
typedef struct gab200_flame_grads {
  float* expr;          /* [T, n_expr] */
  float* rotation;      /* [T, 3] */
  float* neck_pose;     /* [T, 3] */
  float* jaw_pose;      /* [T, 3] */
  float* eyes_pose;     /* [T, 6] */
  float* translation;   /* [T, 3] */
} gab200_flame_grads;
int32_t gab200_flame_backward(const gab200_flame_frame_args* args, const float* dL_dverts, const float* dL_dverts_cano,
                              const gab200_flame_grads* grads, void* stream);

/* Debug/parity access to a finished forward: copies the sorted (key,value) stream and tile ranges to caller
 * DEVICE buffers: keys [N] u64, values [N] u32, ranges [tiles,2] u32. Any may be NULL. */
int32_t gab200_export_binning(const gab200_forward_args* args, const gab200_frame_state* state, uint64_t* keys,
                              uint32_t* values, uint32_t* ranges, void* stream);

/* Opt-in per-stage device timing (profiling aid used by bench.py's roofline line).  When enabled, forward/backward
 * bracket every stage with cudaEvents on the launching stream.  gab200_stage_times() synchronises the pending
 * events, adds them to per-stage totals and returns totals (milliseconds) and launch counts since the last reset. */
enum {
  GAB200_STAGE_PREPROCESS = 0,
  GAB200_STAGE_SCAN = 1,
  GAB200_STAGE_EMIT_KEYS = 2,
  GAB200_STAGE_SORT = 3,
  GAB200_STAGE_TILE_RANGES = 4,
  GAB200_STAGE_BLEND_FWD = 5,
  GAB200_STAGE_BLEND_BWD = 6,
  GAB200_STAGE_PREPROCESS_BWD = 7,
  GAB200_NUM_STAGES = 8
};
void gab200_stage_timing_enable(int32_t enable);
/* Host-side wall time (microseconds, accumulated since the last reset) spent inside gab200_forward, split into
 * [0] launches before the sync, [1] waiting for N, [2] binning allocation callback(s), [3] emit+sort+ranges dispatch,
 * [4] blend dispatch, [5] number of forwards.  Profiling aid; always on (a few clock reads per call). */
void gab200_host_times(double out[6], int32_t reset);
int32_t gab200_stage_times(double total_ms[GAB200_NUM_STAGES], int64_t launches[GAB200_NUM_STAGES], int32_t reset);

/* Tuning knobs (process-wide, atomics; every value has a built-in default that suits the headline workload).
 * gab200_tune(knob, value) sets a knob and returns the previous value; value < 0 only queries. */
enum {
  GAB200_TUNE_HEAVY_FWD = 0,   /* forward blend: a tile is "heavy" (1 px/thread, 8 warps) from this list length (default 32) */
  GAB200_TUNE_HEAVY_BWD = 1,   /* backward blend: a tile is "heavy" (K = 2, 4 warps) from this list length (default 2048) */
  GAB200_TUNE_DEPTH_SORT = 2,  /* 0 (default): bucket sort when a depth hint is given; 1: always cub radix sort */
  GAB200_TUNE_TILE_SORT = 4,   /* per-instance sort by tile: 0 (default) cub::DeviceRadixSort::SortPairs over the instances
                                  (5 launches + tile-range detection); 1 counting sort by tile + per-tile rank sort
                                  (csrc/tile_sort.cu: 3 launches, no memsets).  Identical sorted streams; the counting form
                                  pays same-address atomics on the hot tiles' counters */
  GAB200_TUNE_NVLS_CTAS = 5,   /* gab200_nvls_allreduce: CTAs of 256 threads (0 = default: 64) */
  GAB200_NUM_TUNABLES = 8
};
int32_t gab200_tune(int32_t knob, int32_t value);

/* Number of kernels launched by this library on the calling process so far (bench.py's gpu_launches claim). */
int64_t gab200_launch_count(void);

const char* gab200_status_string(int32_t status);
uint32_t gab200_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GAB200_RASTERIZER_H */
