/*
 * gsraster.h -- C ABI of the H100-native differentiable 3D-Gaussian-Splatting rasterizer.
 *
 * Drop-in boundary for the reference's native rasterizer
 *   RAST = submodules/depth-diff-gaussian-rasterization-min   (LucidDreamer @ 76ed990)
 * Each entry point names the reference interface it replaces.  Plain C: raw device pointers, sizes and
 * scalars; no torch / C++ types.  Every function returns 0 on success or a negative GS_E* code;
 * gs_last_error() returns a human-readable message for the calling thread.
 *
 * The reference's static C++ API (RAST/cuda_rasterizer/rasterizer.h:20-87) takes three
 * std::function<char*(size_t)> "resize" callbacks because the size of the binning buffer is only known
 * after the per-Gaussian pass.  The same two-phase structure is explicit here:
 *
 *   gs_forward_preprocess()  enqueue per-Gaussian pass + tile histogram/scan      (no host sync)
 *   gs_forward_counts()      wait for that pass only; returns num_rendered + #pairs (host sync on an event)
 *   gs_forward_render()      enqueue pair emission + per-tile depth sort + compositing, given a binning
 *                            buffer with room for `pair_capacity` pairs.  If the capacity is too small the
 *                            kernels do nothing (device-side guard) and gs_forward_counts() tells the
 *                            caller how much is needed -> grow and call gs_forward_render() again.
 *
 * A caller may therefore enqueue render() speculatively with the previous frame's capacity *before*
 * calling counts(): the GPU never idles waiting for the host (the reference blocks on a cudaMemcpy D2H
 * every forward, RAST/cuda_rasterizer/rasterizer_impl.cu:282).
 *
 * All work is enqueued on the caller's stream; the library keeps no mutable global state apart from the
 * GsContext (pinned status slots + events), which may be shared by calls on different streams.
 */
#ifndef GSRASTER_H_
#define GSRASTER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GS_ABI_VERSION 2

/* error codes */
#define GS_OK 0
#define GS_EINVAL (-1)   /* bad argument (shape / null pointer / exactly-one-of violated) */
#define GS_ECUDA (-2)    /* CUDA runtime error (message has cudaGetErrorString) */
#define GS_ECAPACITY (-3)/* binning buffer too small: see gs_forward_counts */
#define GS_ENOMEM (-4)
#define GS_ENOTREADY (-5)/* gs_forward_counts_peek: the device has not written the counts yet */

/* status slots of a context and the tickets that name them (gs_forward_preprocess): an eager forward's ticket is
 * slot + GS_STATUS_SLOTS * generation (slots are recycled), a captured forward's is GS_GRAPH_TICKET | its persistent slot */
#define GS_STATUS_SLOTS 64
#define GS_GRAPH_STATUS_SLOTS 256
#define GS_GRAPH_TICKET 0x40000000

typedef struct GsContext GsContext;
typedef void* gs_stream_t; /* cudaStream_t */

/*
 * One view ("frame") of one Gaussian set: the argument list shared by
 * CudaRasterizer::Rasterizer::forward / ::backward (rasterizer.h:35-58, 61-86).
 * Device pointers, float32, contiguous.  NULL = absent, i.e. the reference binding's empty-tensor convention
 * (RAST/depth_diff_gaussian_rasterization_min/__init__.py:198-208): exactly one of shs / colors_precomp and
 * exactly one of (scales & rotations) / cov3D_precomp must be non-NULL.
 */
typedef struct GsFrame {
    int32_t P;               /* #Gaussians */
    int32_t D;               /* active SH degree 0..3 */
    int32_t M;               /* SH coefficients stored per channel (16 at degree 3); 0 if shs == NULL */
    int32_t W, H;            /* image size */
    float tan_fovx, tan_fovy;
    float scale_modifier;
    int32_t prefiltered;     /* accepted for API parity; see DESIGN.md */
    int32_t debug;           /* != 0: synchronize + check after every stage (auxiliary.h:166-173) */
    const float* bg;             /* [3] */
    const float* means3D;        /* [P,3] */
    const float* shs;            /* [P,M,3] or NULL; base pointer 16-byte aligned (128-bit loads) */
    const float* colors_precomp; /* [P,3]   or NULL */
    const float* opacities;      /* [P,1] */
    const float* scales;         /* [P,3]   or NULL */
    const float* rotations;      /* [P,4]   or NULL (r,x,y,z), used un-normalised like forward.cu:127; base pointer
                                    16-byte aligned.  The Python / torch hosts clone misaligned views. */
    const float* cov3D_precomp;  /* [P,6]   or NULL */
    const float* viewmatrix;     /* [16] m[r+4c] = W2C[r][c]        (scene/cameras.py:58) */
    const float* projmatrix;     /* [16] (Proj.W2C), same layout    (scene/cameras.py:60) */
    const float* campos;         /* [3] */
} GsFrame;

/* Gradient outputs of one backward: the tensors RasterizeGaussiansBackwardCUDA returns
 * (RAST/rasterize_points.cu:154-199).  Every non-NULL output is FULLY overwritten (rows of invisible
 * Gaussians get zeros) so the caller may pass uninitialised memory -- no torch::zeros fills needed.
 * NULL = not wanted. */
typedef struct GsGrads {
    float* dL_dmeans3D;   /* [P,3] */
    float* dL_dmeans2D;   /* [P,3]  x,y = dL/d(NDC mean), z = 0 */
    float* dL_dsh;        /* [P,M,3] */
    float* dL_dcolors;    /* [P,3]  gradient w.r.t. colors_precomp (or the SH-derived RGB) */
    float* dL_dopacity;   /* [P,1] */
    float* dL_dscales;    /* [P,3] */
    float* dL_drotations; /* [P,4] */
    float* dL_dcov3D;     /* [P,6] */
    /* Data-parallel shared-model step (no reference counterpart; SURVEY.md 8e).  peer_world > 0: instead of
     * writing dL_dmeans3D / dL_dsh / dL_dopacity / dL_dscales / dL_drotations locally, the final kernel ADDS the rows
     * of this view's visible Gaussians into every rank's gradient bucket: peer_buckets[r] is the (peer-mapped) base
     * of rank r's bucket for r < peer_world (<= 16), peer_multicast optionally the NVSwitch multicast address of the
     * same buckets (then one multimem.red per element replaces peer_world stores), peer_seg_off[5] the float
     * offsets of the five segments inside a bucket.  Buckets must be zeroed and all ranks synchronised before,
     * and synchronised again after, by the caller.  dL_dmeans2D is still written locally. */
    int32_t peer_world;
    int32_t peer_pad;
    void* const* peer_buckets;   /* HOST array of peer_world device pointers */
    void* peer_multicast;
    const int64_t* peer_seg_off; /* HOST array [5] */
    /* Optional cross-rank barriers around the peer adds, run by the library as one-warp kernels (instead of two
     * barriers issued by the host): peer_signals[r] = rank r's signal words (peer-mapped uint32[64], zero-initialised,
     * symmetric), peer_rank = this rank.  peer_epoch_begin != 0: "every rank has cleared its bucket" is awaited before
     * the adds -- gs_backward puts that wait on a side stream beside the tile pass; peer_epoch_end != 0: the call's
     * stream continues only after every rank's adds of this epoch have landed.  Epochs increase by one per
     * optimisation step.  NULL / 0: the caller synchronises the ranks. */
    void* const* peer_signals;   /* HOST array of peer_world device pointers, or NULL */
    int32_t peer_rank;
    uint32_t peer_epoch_begin;
    uint32_t peer_epoch_end;
    int32_t peer_pad2;
} GsGrads;

/* Host-visible result of the per-Gaussian pass. */
typedef struct GsCounts {
    int64_t num_rendered; /* sum of tile-rect areas == the reference's return value (rasterizer_impl.cu:282) */
    int64_t num_pairs;    /* (tile, Gaussian) pairs actually binned (== num_rendered unless culling is on) */
    int64_t num_visible;  /* #{radii > 0} */
} GsCounts;

int gs_abi_version(void);
const char* gs_last_error(void);

/* Context: per device.  Holds pinned status slots + events used by gs_forward_counts. */
int gs_context_create(int device, GsContext** out);
void gs_context_destroy(GsContext* ctx);

/* Scratch sizing -- replaces required<GeometryState/ImageState/BinningState>() (rasterizer_impl.h:66-73).
 * The buffers are opaque to the caller and are what the reference round-trips through
 * ctx.save_for_backward as geomBuffer / binningBuffer / imgBuffer (__init__.py:97). */
size_t gs_geom_bytes(int32_t P);
size_t gs_image_bytes(int32_t W, int32_t H);
size_t gs_binning_bytes(int64_t pair_capacity);

/* replaces the first half of Rasterizer::forward (rasterizer_impl.cu:198-282).
 * radii [P] int32 is fully written.  *ticket identifies the status slot for gs_forward_counts. */
int gs_forward_preprocess(GsContext* ctx, const GsFrame* f, void* geom_buffer, void* image_buffer, int32_t* radii,
                          gs_stream_t stream, int32_t* ticket);

/* Blocks the host until the preprocess of `ticket` has finished (event wait; later work keeps running).
 * A context keeps GS_STATUS_SLOTS status slots: a ticket whose slot has been handed out again (more than GS_STATUS_SLOTS
 * forwards enqueued on the context since) is rejected with GS_EINVAL instead of returning another forward's counts. */
int gs_forward_counts(GsContext* ctx, int32_t ticket, GsCounts* out);

/* Sync-free forward (no reference counterpart: the reference blocks on a D2H copy every forward).  A caller that
 * passes its own `pair_capacity` to gs_forward_render need not call gs_forward_counts at all -- the forward is then
 * pure stream work and can be captured into a CUDA graph (a captured gs_forward_preprocess gets a persistent status
 * slot; at most GS_GRAPH_STATUS_SLOTS alive per context, see gs_forward_release_graph_slot).  If the frame has more pairs than the
 * capacity, the device-side guard renders NOTHING (outputs undefined); the caller finds out here, without blocking:
 * GS_OK + counts once the device has written them (compare counts.num_pairs with the capacity used), GS_ENOTREADY
 * before that.  For a captured forward the slot is rewritten by every replay: synchronise with the replay before
 * trusting it. */
int gs_forward_counts_peek(GsContext* ctx, int32_t ticket, GsCounts* out);

/* Returns the persistent status slot of a captured forward (ticket from gs_forward_preprocess under capture) to the
 * context, so that a process which captures, drops and re-captures graphs (e.g. after every densification) never runs
 * out of the GS_GRAPH_STATUS_SLOTS slots.  Call it only after the graph that holds the forward has been destroyed and no replay of it is
 * pending; the ticket is invalid afterwards (its slot goes to the next capture).  GS_EINVAL for a ticket that is not a
 * captured forward's or whose slot is not in use. */
int gs_forward_release_graph_slot(GsContext* ctx, int32_t ticket);

/* replaces the second half of Rasterizer::forward (rasterizer_impl.cu:284-338).
 * out_color [3,H,W], out_depth [1,H,W] are fully written.  Returns GS_OK even if the capacity turns out
 * too small on the device (nothing is rendered then) -- check with gs_forward_counts.  rerender = 0 for the first
 * render of a frame (it also shades the visible Gaussians), 1 when repeating it with a larger binning buffer. */
int gs_forward_render(GsContext* ctx, const GsFrame* f, const int32_t* radii, void* geom_buffer, void* binning_buffer,
                      int64_t pair_capacity, void* image_buffer, float* out_color, float* out_depth,
                      int32_t rerender, gs_stream_t stream);

/* Batched forward (SURVEY.md 8b "batched variants (n_views, arrays of camera structs)", 8e ">= 2 views in flight"):
 * renders n_views frames (normally the same Gaussians under different cameras: the reference's render_video loop,
 * luciddreamer.py:250-262, or the views of one optimisation step) with up to n_streams views IN FLIGHT on internal
 * streams of the context, forked from and joined back into `stream`.  The reference renders views one by one on
 * the legacy default stream and blocks the host once per view (rasterizer_impl.cu:282); here nothing blocks until
 * every view is enqueued, then the call collects the counts of all views.
 *   scratch[s], s < n_streams (<= 8): geometry / image / binning buffers (+ radii) shared by the views that run on
 *   internal stream s (view k runs on stream k % n_streams; views of one stream are ordered, so they may share).
 *   results[k].out_color / out_depth: per-view outputs ([3,H,W] / [1,H,W]); radii optional (NULL: scratch radii).
 *   results[k].counts and .status are filled on return: GS_OK, or GS_ECAPACITY when the view had more pairs than
 *   scratch[k % n_streams].pair_capacity -- its outputs are then undefined and the caller re-renders that view with
 *   a larger buffer (gs_forward_preprocess / gs_forward_render).  Returns GS_ECAPACITY if any view overflowed. */
typedef struct GsViewScratch {
    void* geom_buffer;      /* gs_geom_bytes(P) */
    void* image_buffer;     /* gs_image_bytes(W, H) */
    void* binning_buffer;   /* gs_binning_bytes(pair_capacity) */
    int64_t pair_capacity;
    int32_t* radii;         /* [P] */
} GsViewScratch;
typedef struct GsViewResult {
    float* out_color;       /* in: [3,H,W] */
    float* out_depth;       /* in: [1,H,W] */
    int32_t* radii;         /* in: [P] or NULL */
    GsCounts counts;        /* out */
    int32_t status;         /* out */
    int32_t pad;
} GsViewResult;
int gs_forward_views(GsContext* ctx, const GsFrame* frames, int32_t n_views, const GsViewScratch* scratch,
                     int32_t n_streams, GsViewResult* results, gs_stream_t stream);

/* replaces Rasterizer::backward (rasterizer_impl.cu:343-444) + the nine torch::zeros of its binding.
 * dL_dout_depth is accepted and ignored: the reference's depth gradient is commented out
 * (backward.cu:443-469,539-554).  When all six of dL_dmeans3D / dL_dmeans2D / dL_dsh (M = 16) / dL_dopacity /
 * dL_dscales / dL_drotations are wanted (bases 16-byte aligned, P a multiple of 4, no peer reduce), the outputs are
 * zero-filled on a side stream of the context beside the tile pass and the per-Gaussian pass writes only the rows of
 * the visible Gaussians. */
size_t gs_backward_scratch_bytes(int64_t num_visible);   /* num_visible from gs_forward_counts (or P as a bound) */
int gs_backward(GsContext* ctx, const GsFrame* f, const int32_t* radii, const void* geom_buffer,
                const void* binning_buffer, int64_t pair_capacity, const void* image_buffer, void* grad_scratch,
                size_t grad_scratch_bytes, const float* dL_dout_color, const float* dL_dout_depth,
                const GsGrads* grads, gs_stream_t stream);

/* Deterministic backward (no reference counterpart: the reference sums every (pixel, splat) partial with float
 * atomics).  Same arguments, outputs and stages as gs_backward, except that each Gaussian's per-tile partials are summed
 * in a fixed order (ascending position in the forward's depth-sorted pair list) instead of by float atomics in
 * completion order: the gradients of one forward are bit-identical from run to run, independent of scheduling, stream
 * concurrency, CUDA-graph replay and the pair capacity.  They agree with gs_backward's up to the order of those float
 * additions.  grad_scratch must hold gs_backward_deterministic_scratch_bytes(num_visible, pair_capacity) bytes
 * (num_visible from gs_forward_counts, or P as a bound; pair_capacity as passed to gs_forward_render).  The peer reduce
 * is not supported: peer_world > 0 returns GS_EINVAL.  Pure stream work, capturable like gs_backward. */
size_t gs_backward_deterministic_scratch_bytes(int64_t num_visible, int64_t pair_capacity);
int gs_backward_deterministic(GsContext* ctx, const GsFrame* f, const int32_t* radii, const void* geom_buffer,
                              const void* binning_buffer, int64_t pair_capacity, const void* image_buffer,
                              void* grad_scratch, size_t grad_scratch_bytes, const float* dL_dout_color,
                              const float* dL_dout_depth, const GsGrads* grads, gs_stream_t stream);

/* replaces Rasterizer::markVisible (rasterizer_impl.cu:141-153): present[i] = (z_view > 0.2) */
int gs_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    uint8_t* present, gs_stream_t stream);

/* "Next" row (SURVEY.md 8f-1), first slice: fused L1 photometric loss + gradient.  Replaces utils/loss.py:18
 * `l1_loss` and its autograd backward in the training step (luciddreamer.py:301-304): loss[0] = weight *
 * mean|color - target/255|, dL_dcolor = weight * sign(color - target/255) / (3HW).  color, dL_dcolor: [3,H,W] f32;
 * target_u8: [H,W,3] uint8 (the layout images arrive in from the host). */
int gs_l1_loss_backward(GsContext* ctx, const float* color, const uint8_t* target_u8, int32_t H, int32_t W, float weight,
                        float* dL_dcolor, float* loss, gs_stream_t stream);

/* "Next" row (SURVEY.md 8f-2): fused optimiser step.  One launch replaces the autograd backward through the parameter
 * activations of scene/gaussian_model.py:97-117 and torch.optim.Adam(eps=1e-15) over the parameter groups of
 * gaussian_model.py:156-165.  `grad` is the gradient w.r.t. the ACTIVATED value as written by gs_backward (e.g. a
 * segment of the flat gradient bucket): the parameter at (row, c) reads grad[row * grad_row_width + grad_offset + c].
 * activation: 0 none (xyz, SH features), 1 sigmoid (opacity logit), 2 exp (log scale), 3 F.normalize (quaternion rows
 * of 4; row_width ignored).  param / exp_avg / exp_avg_sq (16-byte aligned) are updated in place; `step` is the 1-based Adam step. */
typedef struct GsAdamGroup {
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    int64_t rows;
    int32_t row_width;
    int32_t grad_row_width;
    int32_t grad_offset;
    int32_t activation;
    double lr;
} GsAdamGroup;
int gs_gaussian_adam_step(GsContext* ctx, const GsAdamGroup* groups, int32_t ngroups, double beta1, double beta2,
                          double eps, int32_t step, gs_stream_t stream);

/* Training step as pure stream work (no reference counterpart; the reference runs these as torch ops).  Every entry point
 * below is capturable in a CUDA graph; bad sizes, NULL or misaligned pointers return GS_EINVAL before any device work.
 *
 * gs_activate: what render() computes from the raw parameters (gaussian_renderer/__init__.py:53-80,
 * scene/gaussian_model.py:97-117), in one launch:
 *   shs = cat(features_dc [P,1,3], features_rest [P,M-1,3]) -> [P,M,3];  opacities = sigmoid(opacity) [P,1];
 *   scales = exp(scaling) [P,3];  rotations = F.normalize(rotation [P,4], dim=1, eps=1e-12) [P,4]
 * Outputs are bit-identical to torch.cat / torch.sigmoid / torch.exp / F.normalize on the device (DESIGN.md).
 * rotation, shs and rotations 16-byte aligned, the rest 4-byte aligned; features_rest may be NULL when M == 1. */
int gs_activate(GsContext* ctx, int32_t P, int32_t M, const float* features_dc, const float* features_rest,
                const float* opacity, const float* scaling, const float* rotation, float* shs, float* opacities,
                float* scales, float* rotations, gs_stream_t stream);

/* Scheduled Adam: gs_gaussian_adam_step's update and activation chain rule, with every per-step scalar read from device
 * memory, so that a CUDA-graph replay steps like an eager call.
 *   step (per group, device float32, torch's state["step"]): advanced by one per executed step; the bias corrections of
 *        step s are bias_bc1[min(s, bias_len-1)] and bias_bc2_sqrt[min(s, bias_len-1)] (gs_adam_bias_table)
 *   lr: lr_table[clamp(*iteration, 0, lr_table_len-1)] when lr_table != NULL, else the host value lr
 *   step_size = (float)(lr / bias_bc1[s]), one IEEE double division on the device; given the same lr and step the
 *   update is bit-identical to gs_gaussian_adam_step.
 * Guard: image_buffer = the forward's image buffer (W x H, rendered with pair_capacity) or NULL.  If that frame had more
 * pairs than pair_capacity, nothing is written: parameters, moments and step counters keep every byte.
 * scratch: gs_adam_sched_scratch_bytes() bytes of device memory, 16-byte aligned, private to the call until it ends. */
typedef struct GsAdamSchedGroup {
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    int64_t rows;
    int32_t row_width;
    int32_t grad_row_width;
    int32_t grad_offset;
    int32_t activation;       /* as GsAdamGroup */
    double lr;                /* used when lr_table == NULL */
    const double* lr_table;   /* device [lr_table_len] or NULL */
    float* step;              /* device float32 scalar, 4-byte aligned */
} GsAdamSchedGroup;
size_t gs_adam_sched_scratch_bytes(void);
/* Length of the bias-correction table for (beta1, beta2): one past the first step at which both corrections are exactly
 * 1 (every later step uses that last entry).  0 if the betas are outside [0, 1) or the table would exceed 2^24 entries. */
int32_t gs_adam_bias_table_len(double beta1, double beta2);
/* Fills HOST arrays bc1[s] = 1 - beta1^s (double) and bc2_sqrt[s] = (float)sqrt(1 - beta2^s) for s < n, formed like
 * gs_gaussian_adam_step forms them (entry 0 is never read). */
int gs_adam_bias_table(double beta1, double beta2, int32_t n, double* bc1, float* bc2_sqrt);
int gs_gaussian_adam_sched_step(GsContext* ctx, const GsAdamSchedGroup* groups, int32_t ngroups, double beta1,
                                double beta2, double eps, const double* bias_bc1, const float* bias_bc2_sqrt,
                                int32_t bias_len, const int32_t* iteration, int32_t lr_table_len,
                                const void* image_buffer, int32_t W, int32_t H, int64_t pair_capacity, void* scratch,
                                size_t scratch_bytes, gs_stream_t stream);

/* gs_densify_stats behind the same guard: if the forward of image_buffer (W x H, pair_capacity) overflowed, the three
 * accumulators keep every byte.  image_buffer = NULL: no guard. */
int gs_densify_stats_guarded(GsContext* ctx, int32_t P, const int32_t* radii, const float* dL_dmeans2D,
                             float* xyz_gradient_accum, float* denom, float* max_radii2D, const void* image_buffer,
                             int32_t W, int32_t H, int64_t pair_capacity, gs_stream_t stream);

/* "Next" row (SURVEY.md 8f-4): per-frame host work of render_video (luciddreamer.py:250-262) moved to the device.
 *   rgb8[y][x][c]  = uint8(round_half_even(clip(color[c][y][x], 0, 1) * 255))           (:254-255)
 *   neg_depth[y][x] = -(depth[y][x] * (depth[y][x] > 0))                                 (:256)
 *   minmax_state   = running {min, max} of neg_depth over all frames packed so far       (:257-262); two uint32 the
 *                    caller initialises to {0xffffffff, 0}; gs_minmax_read decodes them to two floats (device).
 * color: [3,H,W] f32; depth: [1,H,W] f32 or NULL (colour only); rgb8: [H,W,3] u8; neg_depth: [H,W] f32. */
int gs_pack_frame(GsContext* ctx, int32_t H, int32_t W, const float* color, const float* depth, uint8_t* rgb8,
                  float* neg_depth, uint32_t* minmax_state, gs_stream_t stream);
int gs_minmax_read(GsContext* ctx, uint32_t* minmax_state, float* minmax2, gs_stream_t stream);

/* Depth colour mapping of a clip: `depthlist = [colorize(depth) for depth in depthlist]` (luciddreamer.py:267,
 * utils/depth.py:7-62 with cmap 'jet'), for F frames in one fixed sequence of launches.  Per frame, over the valid pixels
 * (value != invalid_val):
 *   vmin, vmax = np.percentile(valid, 2), np.percentile(valid, 98)   evaluated as numpy does for float32 input
 *                (float32 index (n-1) * float32(q/100), float32 lerp), from exact order statistics (radix select)
 *   x = (value - vmin) / (vmax - vmin)  (IEEE float32) if vmin != vmax, else 0
 *   rgba[y][x] = lut_rgba[clamp(trunc(x * 256), 0, 255)] (x < 0 -> entry 0, x > 1 -> entry 255); invalid pixels get
 *                background_rgba (bytes R, G, B, A in memory order, i.e. R | G << 8 | B << 16 | A << 24)
 * The result is bit-identical to the host restatement (luciddreamer_b200.video.colorize) on the same float32 frame.
 * A frame without a valid pixel (where np.percentile raises) is all background and gets NaN for its (vmin, vmax).
 * -0.0 and +0.0 count as one value; NaN / inf depths are outside the contract (every output byte is still written).
 *   value: [F,H,W] f32 device; lut_rgba: [256,4] u8 device; rgba: [F,H,W,4] u8 device; all 4-byte aligned
 *   vminmax: [F,2] f32 device, or NULL;  scratch: gs_colorize_scratch_bytes(F) bytes, 16-byte aligned
 * Pure stream work (capturable in a CUDA graph).  ctx is not used and may be NULL. */
size_t gs_colorize_scratch_bytes(int32_t F);
int gs_colorize_depth(GsContext* ctx, int32_t F, int32_t H, int32_t W, const float* value, float invalid_val,
                      const uint8_t* lut_rgba, uint32_t background_rgba, void* scratch, size_t scratch_bytes,
                      uint8_t* rgba, float* vminmax, gs_stream_t stream);

/* "Next" row (SURVEY.md 8f-3): simple_knn.distCUDA2 (submodules/simple-knn/spatial.cu:15-26 over SimpleKNN::knn,
 * simple_knn.cu:185-221): mean_dist2[i] = mean of the squared distances from point i to its 3 nearest other points
 * (exact search; bit-identical to the reference, incl. duplicates and P < 4).  points: [P,3] f32 device;
 * scratch: gs_knn_scratch_bytes(P) bytes, 256-byte aligned; mean_dist2: [P] f32 device. */
size_t gs_knn_scratch_bytes(int32_t P);
int gs_knn_mean_dist2(GsContext* ctx, int32_t P, const float* points, void* scratch, float* mean_dist2, gs_stream_t stream);

/* Densification statistics of one view (luciddreamer.py:308-312, scene/gaussian_model.py:405-407), one pass: for every
 * Gaussian with radii > 0:  max_radii2D = max(max_radii2D, radii);  xyz_gradient_accum += ||dL_dmeans2D[:, :2]||;
 * denom += 1.  radii: [P] int32; dL_dmeans2D: [P,3]; the three accumulators: [P] f32 (in place). */
int gs_densify_stats(GsContext* ctx, int32_t P, const int32_t* radii, const float* dL_dmeans2D, float* xyz_gradient_accum,
                     float* denom, float* max_radii2D, gs_stream_t stream);

/* "Next" row (SURVEY.md 8f-1): the reference's full photometric training loss and its gradient, fused:
 *   loss3[0] = (1 - lambda) * l1_loss(image, gt) + lambda * (1 - ssim(image, gt))     (luciddreamer.py:301-303)
 *   loss3[1] = l1_loss (utils/loss.py:18),  loss3[2] = ssim (utils/loss.py:38-69: 11x11 Gaussian window, sigma 1.5,
 *   zero padding, C1 = 0.01^2, C2 = 0.03^2, mean over all elements)
 *   dL_dimage = d loss3[0] / d image   (NULL: forward only)
 * image, gt, dL_dimage: [3,H,W] f32 device; loss3: [3] f32 device; scratch: gs_photometric_scratch_bytes(H, W). */
size_t gs_photometric_scratch_bytes(int32_t H, int32_t W);
int gs_photometric_loss_backward(GsContext* ctx, const float* image, const float* gt, int32_t H, int32_t W,
                                 float lambda_dssim, void* scratch, float* dL_dimage, float* loss3, gs_stream_t stream);

/* Introspection for tests: copies the per-tile exclusive offsets (uint32 [G+1]; tile t owns
 * [off[t], off[t+1]) -- the reference's `ranges`, rasterizer_impl.cu:116-138) and the depth-sorted Gaussian
 * index list (uint32 [max_pairs]; the reference's `point_list`) out of the opaque buffers (device -> device). */
int gs_debug_export_binning(const GsFrame* f, const void* binning_buffer, int64_t pair_capacity,
                            const void* image_buffer, uint32_t* tile_offsets, uint32_t* point_list,
                            int64_t max_pairs, gs_stream_t stream);

/* Introspection for tests: the image rows a warp of the tile passes (forward blend, backward, deterministic partials)
 * owns when a W x H frame is rendered on ctx's device: 4 (16x4 strips, four warps per tile) or 8 (16x8 blocks, two
 * warps).  The choice depends on the tile count and the device's SM count; this asks the launch code itself.
 * Negative on a bad argument. */
int gs_debug_blend_rows_per_warp(GsContext* ctx, int32_t W, int32_t H);

/* Per-kernel timing for bench.py's roofline leg (no reference counterpart: the reference has no profiling hooks,
 * SURVEY.md section 5).  When enabled, every kernel launch is bracketed by CUDA events on the launching stream;
 * gs_profile_read waits for them and returns the duration in ms of each kernel of the most recent forward /
 * backward (-1 = not launched).  Kernel i is named gs_profile_kernel_name(i), i < gs_profile_num_kernels(). */
#define GS_NUM_KERNELS 12
int gs_profile_enable(GsContext* ctx, int on);
int gs_profile_num_kernels(void);
const char* gs_profile_kernel_name(int i);
int gs_profile_read(GsContext* ctx, float* ms);

#ifdef __cplusplus
}
#endif
#endif /* GSRASTER_H_ */
