// C ABI of the H100 rasterizer (include/gsraster.h).  Host-side orchestration only: argument checks, scratch
// carving, kernel launches on the caller's stream, pinned status slots.  Mirrors the structure of the
// reference's CudaRasterizer::Rasterizer::{forward,backward,markVisible}
// (RAST/cuda_rasterizer/rasterizer_impl.cu:141-153,198-339,343-444) and of its torch binding
// (RAST/rasterize_points.cu:35-221) without any torch types.
#include <atomic>
#include <mutex>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../include/gsraster.h"
#include "gs_common.cuh"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define GS_CUDA(expr)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (expr);                                                                        \
        if (e_ != cudaSuccess) return fail(GS_ECUDA, "%s failed: %s", #expr, cudaGetErrorString(e_));   \
    } while (0)

constexpr int kMaxViewStreams = 8;

int check_frame(const GsFrame* f) {
    if (!f) return fail(GS_EINVAL, "frame is NULL");
    if (f->P < 0 || f->W <= 0 || f->H <= 0) return fail(GS_EINVAL, "bad sizes P=%d W=%d H=%d", f->P, f->W, f->H);
    if (f->P == 0) return GS_OK;
    if (!f->means3D || !f->opacities || !f->viewmatrix || !f->projmatrix || !f->campos || !f->bg)
        return fail(GS_EINVAL, "means3D/opacities/viewmatrix/projmatrix/campos/bg must be non-NULL");
    // RAST/depth_diff_gaussian_rasterization_min/__init__.py:192-196
    if ((f->shs == nullptr) == (f->colors_precomp == nullptr))
        return fail(GS_EINVAL, "Please provide excatly one of either SHs or precomputed colors!");
    if (((f->scales == nullptr || f->rotations == nullptr) && f->cov3D_precomp == nullptr) ||
        ((f->scales != nullptr || f->rotations != nullptr) && f->cov3D_precomp != nullptr))
        return fail(GS_EINVAL, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    // k_project / k_grad_vis / sh_to_rgb read rotations and SH rows with 128-bit loads
    if ((reinterpret_cast<uintptr_t>(f->rotations) & 15) || (reinterpret_cast<uintptr_t>(f->shs) & 15))
        return fail(GS_EINVAL, "rotations and shs must be 16-byte aligned (see gsraster.h)");
    if (f->shs && (f->M <= 0 || f->D < 0 || f->D > 3 || (f->D + 1) * (f->D + 1) > f->M))
        return fail(GS_EINVAL, "SH degree %d needs %d coefficients, M=%d", f->D, (f->D + 1) * (f->D + 1), f->M);
    return GS_OK;
}

GsView make_view(const GsFrame* f) {
    GsView v;
    v.vm = f->viewmatrix; v.pm = f->projmatrix; v.campos = f->campos; v.bg = f->bg;
    v.tan_fovx = f->tan_fovx; v.tan_fovy = f->tan_fovy;
    v.focal_y = f->H / (2.0f * f->tan_fovy);            // rasterizer_impl.cu:223-224
    v.focal_x = f->W / (2.0f * f->tan_fovx);
    v.scale_modifier = f->scale_modifier;
    v.W = f->W; v.H = f->H;
    v.gx = (f->W + GS_TILE - 1) / GS_TILE; v.gy = (f->H + GS_TILE - 1) / GS_TILE;
    v.P = f->P; v.D = f->D; v.M = f->shs ? f->M : 0;
    return v;
}

int debug_sync(const GsFrame* f, cudaStream_t s, const char* what) {
    if (!f->debug) {
        cudaError_t e = cudaPeekAtLastError();
        if (e != cudaSuccess) return fail(GS_ECUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
        return GS_OK;
    }
    cudaError_t e = cudaStreamSynchronize(s);           // CHECK_CUDA(., debug): auxiliary.h:166-173
    if (e != cudaSuccess) return fail(GS_ECUDA, "[CUDA ERROR] in %s: %s", what, cudaGetErrorString(e));
    return GS_OK;
}

}  // namespace

__global__ void k_clear_words(uint32_t* __restrict__ p, size_t words) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) p[i] = 0u;
}
void gs_launch_clear_words(uint32_t* p, size_t words, cudaStream_t s) {
    if (!words) return;
    const int grid = (int)((words + 255) / 256 < 296 ? (words + 255) / 256 : 296);
    k_clear_words<<<grid, 256, 0, s>>>(p, words);
}

constexpr int kNumKernels = GS_NUM_KERNELS;
static const char* const kKernelNames[kNumKernels] = {"k_project", "k_tile_scan", "k_shade_emit", "k_tile_sort",
                                                      "k_tile_sort_big", "k_blend_fwd", "k_blend_bwd", "k_grad_vis",
                                                      "k_count_tiles", "k_grad_write",   // slot 9 also times
                                                      "k_grad_dense", "k_fill_zero"};    // k_grad_reduce_peers

struct GsContext {
    int device;
    int num_sms;
    int profile;                   // != 0: bracket every kernel with timing events (gs_profile_*)
    cudaEvent_t pev[2 * kNumKernels];
    bool pev_used[kNumKernels];
    GsDevStatus* slots;            // pinned, mapped: GS_STATUS_SLOTS recycled slots, then GS_GRAPH_STATUS_SLOTS persistent ones
    std::mutex graph_mu;           // guards graph_used
    bool graph_used[GS_GRAPH_STATUS_SLOTS];  // persistent slot owned by a captured forward until it is released
    std::atomic<long long> last_visible;   // num_visible of the most recent forward whose counts were read (-1: none yet)
    cudaEvent_t events[GS_STATUS_SLOTS];
    unsigned slot_gen[GS_STATUS_SLOTS];     // generation of the ticket that currently owns the slot
    std::atomic<unsigned> next;
    cudaStream_t aux;              // side stream of gs_backward's zero-fill (beside the tile pass) and peer barrier
    cudaEvent_t aux_fork, aux_join;
    bool aux_ready;
    cudaStream_t vstreams[kMaxViewStreams];   // internal streams of gs_forward_views (created on first use)
    cudaEvent_t vfork, vjoin[kMaxViewStreams];
    bool vstreams_ready;
};

// Brackets a launch with timing events on the launching stream when profiling is on (bench.py's roofline leg).
#define GS_TIMED(ctx, k, s, launch)                                   \
    do {                                                              \
        if ((ctx) && (ctx)->profile) cudaEventRecord((ctx)->pev[2 * (k)], s);     \
        launch;                                                       \
        if ((ctx) && (ctx)->profile) { cudaEventRecord((ctx)->pev[2 * (k) + 1], s); (ctx)->pev_used[k] = true; } \
    } while (0)

extern "C" {

int gs_profile_enable(GsContext* ctx, int on) {
    if (!ctx) return fail(GS_EINVAL, "ctx is NULL");
    ctx->profile = on;
    for (int i = 0; i < kNumKernels; i++) ctx->pev_used[i] = false;
    return GS_OK;
}
int gs_profile_num_kernels(void) { return kNumKernels; }
const char* gs_profile_kernel_name(int i) { return (i >= 0 && i < kNumKernels) ? kKernelNames[i] : ""; }
int gs_profile_read(GsContext* ctx, float* ms) {
    if (!ctx || !ms) return fail(GS_EINVAL, "NULL argument");
    for (int k = 0; k < kNumKernels; k++) {
        ms[k] = -1.f;
        if (!ctx->pev_used[k]) continue;
        GS_CUDA(cudaEventSynchronize(ctx->pev[2 * k + 1]));
        GS_CUDA(cudaEventElapsedTime(&ms[k], ctx->pev[2 * k], ctx->pev[2 * k + 1]));
    }
    return GS_OK;
}

int gs_abi_version(void) { return GS_ABI_VERSION; }
const char* gs_last_error(void) { return g_err; }

int gs_context_create(int device, GsContext** out) {
    if (!out) return fail(GS_EINVAL, "out is NULL");
    int prev = 0;
    GS_CUDA(cudaGetDevice(&prev));
    GS_CUDA(cudaSetDevice(device));
    GsContext* c = new GsContext();
    c->device = device;
    c->next = 0;
    for (int i = 0; i < GS_GRAPH_STATUS_SLOTS; i++) c->graph_used[i] = false;
    c->last_visible = -1;
    c->profile = 0;
    c->vstreams_ready = false;
    c->aux_ready = false;
    for (int i = 0; i < GS_STATUS_SLOTS; i++) c->slot_gen[i] = 0;
    for (int i = 0; i < kNumKernels; i++) c->pev_used[i] = false;
    for (int i = 0; i < 2 * kNumKernels; i++) cudaEventCreate(&c->pev[i]);
    c->num_sms = g_gs_num_sms;
    cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device);
    g_gs_num_sms = c->num_sms;
    gs_tile_sort_init();
    gs_det_bwd_init();
    gs_grad_write_init();
    gs_preprocess_init();
    cudaError_t e = cudaHostAlloc((void**)&c->slots, sizeof(GsDevStatus) * (GS_STATUS_SLOTS + GS_GRAPH_STATUS_SLOTS),
                                cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) {
        for (int j = 0; j < 2 * kNumKernels; j++) cudaEventDestroy(c->pev[j]);
        delete c;
        cudaSetDevice(prev);
        return fail(GS_ECUDA, "cudaHostAlloc: %s", cudaGetErrorString(e));
    }
    memset(c->slots, 0, sizeof(GsDevStatus) * (GS_STATUS_SLOTS + GS_GRAPH_STATUS_SLOTS));
    for (int i = 0; i < GS_STATUS_SLOTS; i++) {
        e = cudaEventCreateWithFlags(&c->events[i], cudaEventDisableTiming);
        if (e != cudaSuccess) {
            for (int j = 0; j < i; j++) cudaEventDestroy(c->events[j]);
            for (int j = 0; j < 2 * kNumKernels; j++) cudaEventDestroy(c->pev[j]);
            cudaFreeHost(c->slots);
            delete c;
            cudaSetDevice(prev);
            return fail(GS_ECUDA, "cudaEventCreate: %s", cudaGetErrorString(e));
        }
    }
    cudaSetDevice(prev);
    *out = c;
    return GS_OK;
}

void gs_context_destroy(GsContext* c) {
    if (!c) return;
    for (int i = 0; i < GS_STATUS_SLOTS; i++) cudaEventDestroy(c->events[i]);
    for (int i = 0; i < 2 * kNumKernels; i++) cudaEventDestroy(c->pev[i]);
    if (c->aux_ready) { cudaEventDestroy(c->aux_fork); cudaEventDestroy(c->aux_join); cudaStreamDestroy(c->aux); }
    if (c->vstreams_ready) {
        cudaEventDestroy(c->vfork);
        for (int i = 0; i < kMaxViewStreams; i++) { cudaEventDestroy(c->vjoin[i]); cudaStreamDestroy(c->vstreams[i]); }
    }
    cudaFreeHost(c->slots);
    delete c;
}

size_t gs_geom_bytes(int32_t P) { return gs_geom_layout(nullptr, P > 0 ? P : 1).bytes; }
size_t gs_image_bytes(int32_t W, int32_t H) { return gs_image_layout(nullptr, W, H).bytes; }
size_t gs_binning_bytes(int64_t cap) { return gs_bin_layout(nullptr, cap > 0 ? cap : 1).bytes; }

// Hands a new forward its status slot (*slot indexes ctx->slots) and the ticket that names it (gsraster.h), and clears
// the slot.  A forward that is being captured into a CUDA graph gets a PERSISTENT slot (the graph bakes its address in
// and rewrites it on every replay); no event is involved, nothing may block.  Eager forwards recycle GS_STATUS_SLOTS slots.
static int acquire_slot(GsContext* ctx, bool capturing, int* slot, int32_t* ticket) {
    if (capturing) {
        int gsl = -1;
        {
            std::lock_guard<std::mutex> lock(ctx->graph_mu);
            for (int i = 0; i < GS_GRAPH_STATUS_SLOTS && gsl < 0; i++)
                if (!ctx->graph_used[i]) { ctx->graph_used[i] = true; gsl = i; }
        }
        if (gsl < 0)
            return fail(GS_ENOMEM, "more than %d forwards captured into CUDA graphs on this context are alive (release the "
                                   "slots of destroyed graphs with gs_forward_release_graph_slot)", GS_GRAPH_STATUS_SLOTS);
        *slot = GS_STATUS_SLOTS + gsl;
        *ticket = GS_GRAPH_TICKET | gsl;
    } else {
        const unsigned seq = ctx->next.fetch_add(1u);
        *slot = (int)(seq % (unsigned)GS_STATUS_SLOTS);
        const unsigned gen = (seq / (unsigned)GS_STATUS_SLOTS) & 0x00ffffffu;     // stays below GS_GRAPH_TICKET
        // the slot's previous owner (GS_STATUS_SLOTS forwards ago) must have written its status before it is cleared
        if (seq >= (unsigned)GS_STATUS_SLOTS) GS_CUDA(cudaEventSynchronize(ctx->events[*slot]));
        ctx->slot_gen[*slot] = gen;
        *ticket = (int32_t)(gen * GS_STATUS_SLOTS + (unsigned)*slot);
    }
    ctx->slots[*slot].overflow = 0;                      // cleared; kernel writes 0xC0FFEE when done
    return GS_OK;
}

int gs_forward_preprocess(GsContext* ctx, const GsFrame* f, void* geom_buffer, void* image_buffer, int32_t* radii,
                          gs_stream_t stream, int32_t* ticket) {
    if (!ctx || !ticket) return fail(GS_EINVAL, "ctx/ticket is NULL");
    int rc = check_frame(f);
    if (rc) return rc;
    if (!image_buffer || (f->P > 0 && (!geom_buffer || !radii))) return fail(GS_EINVAL, "scratch/radii is NULL");
    cudaStream_t s = (cudaStream_t)stream;
    const GsView v = make_view(f);
    const int G = v.gx * v.gy;
    GsImageLayout il = gs_image_layout(image_buffer, f->W, f->H);
    cudaStreamCaptureStatus cap_st = cudaStreamCaptureStatusNone;
    GS_CUDA(cudaStreamIsCapturing(s, &cap_st));
    const bool capturing = cap_st != cudaStreamCaptureStatusNone;
    int slot = -1;
    if ((rc = acquire_slot(ctx, capturing, &slot, ticket))) return rc;
    // zero tile histogram + status in one memset (they are adjacent)
    gs_launch_clear_words(il.tile_cnt, ((size_t)((char*)il.status - (char*)il.tile_cnt) + sizeof(GsDevStatus)) / 4, s);
    GsDevStatus* dev_slot = nullptr;
    GS_CUDA(cudaHostGetDevicePointer((void**)&dev_slot, ctx->slots + slot, 0));
    if (f->P > 0) {
        GsGeomLayout gl = gs_geom_layout(geom_buffer, f->P);
        GS_TIMED(ctx, 0, s, gs_launch_project(v, f->means3D, f->opacities, f->scales, f->rotations, f->cov3D_precomp,
                                              radii, gl.rec, gl.vis_list, il.status,
                                              2 * ctx->last_visible.load() > (long long)f->P, s));
        if ((rc = debug_sync(f, s, "project"))) return rc;
        // the tile histogram; its last CTA also scans it and mirrors the totals to the host slot
        GS_TIMED(ctx, 8, s, gs_launch_count_tiles(v, ctx->num_sms, radii, gl.rec, gl.vis_list, gl.hitmask, il.tile_cnt, il.status,
                                                  il.tile_off, dev_slot, s));
        if ((rc = debug_sync(f, s, "count_tiles"))) return rc;
    } else {                                             // no Gaussians: k_count_tiles does not run, scan the empty histogram
        GS_TIMED(ctx, 1, s, gs_launch_tile_scan(G, il.tile_cnt, il.tile_off, il.status, dev_slot, s));
        if ((rc = debug_sync(f, s, "tile_scan"))) return rc;
    }
    if (!capturing) GS_CUDA(cudaEventRecord(ctx->events[slot], s));
    return GS_OK;
}

static int read_slot(GsContext* ctx, int slot, GsCounts* out, bool must_be_ready) {
    const volatile GsDevStatus* h = ctx->slots + slot;
    if (h->overflow != 0xC0FFEEu) {
        if (must_be_ready) return fail(GS_ECUDA, "status slot %d was not written by the device", slot);
        return GS_ENOTREADY;
    }
    out->num_rendered = (int64_t)h->num_rendered;
    out->num_pairs = (int64_t)h->num_pairs;
    out->num_visible = (int64_t)h->num_visible;
    ctx->last_visible = out->num_visible;
    return GS_OK;
}

// The status slot (index into ctx->slots) that a non-negative ticket names (gsraster.h).  GS_EINVAL for a captured
// forward's slot out of range, or an eager ticket whose slot has been handed to a later forward.
static int ticket_slot(const GsContext* ctx, int32_t ticket, int* slot) {
    if (ticket & GS_GRAPH_TICKET) {
        const int gsl = ticket & (GS_GRAPH_TICKET - 1);
        if (gsl >= GS_GRAPH_STATUS_SLOTS) return fail(GS_EINVAL, "bad graph ticket");
        *slot = GS_STATUS_SLOTS + gsl;
        return GS_OK;
    }
    *slot = ticket % GS_STATUS_SLOTS;
    if (ctx->slot_gen[*slot] == (unsigned)ticket / GS_STATUS_SLOTS) return GS_OK;
    return fail(GS_EINVAL, "ticket expired: more than %d forwards were enqueued on this context since", GS_STATUS_SLOTS);
}

int gs_forward_counts(GsContext* ctx, int32_t ticket, GsCounts* out) {
    if (!ctx || !out || ticket < 0) return fail(GS_EINVAL, "bad ctx/ticket/out");
    if (ticket & GS_GRAPH_TICKET)
        return fail(GS_EINVAL, "ticket of a captured forward: replay the graph, synchronise, then gs_forward_counts_peek");
    int slot, rc;
    if ((rc = ticket_slot(ctx, ticket, &slot))) return rc;
    GS_CUDA(cudaEventSynchronize(ctx->events[slot]));
    if ((rc = ticket_slot(ctx, ticket, &slot))) return rc;      // the slot may have been handed out during the wait
    return read_slot(ctx, slot, out, true);
}

int gs_forward_release_graph_slot(GsContext* ctx, int32_t ticket) {
    if (!ctx || ticket < 0 || !(ticket & GS_GRAPH_TICKET)) return fail(GS_EINVAL, "not the ticket of a captured forward");
    int slot;
    const int rc = ticket_slot(ctx, ticket, &slot);
    if (rc) return rc;
    const int gsl = slot - GS_STATUS_SLOTS;
    std::lock_guard<std::mutex> lock(ctx->graph_mu);
    if (!ctx->graph_used[gsl]) return fail(GS_EINVAL, "graph status slot %d is not in use (released twice?)", gsl);
    memset((void*)(ctx->slots + slot), 0, sizeof(GsDevStatus));     // a stale peek now reads "not ready"
    ctx->graph_used[gsl] = false;
    return GS_OK;
}

int gs_forward_counts_peek(GsContext* ctx, int32_t ticket, GsCounts* out) {
    if (!ctx || !out || ticket < 0) return fail(GS_EINVAL, "bad ctx/ticket/out");
    int slot;
    const int rc = ticket_slot(ctx, ticket, &slot);
    return rc ? rc : read_slot(ctx, slot, out, false);
}

int gs_forward_render(GsContext* ctx, const GsFrame* f, const int32_t* radii, void* geom_buffer, void* binning_buffer,
                      int64_t pair_capacity, void* image_buffer, float* out_color, float* out_depth,
                      int32_t rerender, gs_stream_t stream) {
    int rc = check_frame(f);
    if (rc) return rc;
    if (!image_buffer || !out_color || !out_depth) return fail(GS_EINVAL, "image buffer / outputs are NULL");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t N = (size_t)f->W * f->H;
    if (f->P == 0) {                                     // rasterize_points.cu:68-70,82: zero images, no kernels
        GS_CUDA(cudaMemsetAsync(out_color, 0, 3 * N * sizeof(float), s));
        GS_CUDA(cudaMemsetAsync(out_depth, 0, N * sizeof(float), s));
        return GS_OK;
    }
    if (!geom_buffer || !radii || !binning_buffer || pair_capacity < 0) return fail(GS_EINVAL, "scratch/radii is NULL");
    const GsView v = make_view(f);
    const int G = v.gx * v.gy;
    GsImageLayout il = gs_image_layout(image_buffer, f->W, f->H);
    GsGeomLayout gl = gs_geom_layout(geom_buffer, f->P);
    GsBinLayout bl = gs_bin_layout(binning_buffer, pair_capacity > 0 ? pair_capacity : 1);
    GS_TIMED(ctx, 2, s, gs_launch_shade_emit(v, ctx ? ctx->num_sms : g_gs_num_sms, f->means3D, f->shs, f->colors_precomp, radii,
                                             gl.rec, gl.acc, gl.vis_list, gl.hitmask, il.tile_off, il.tile_cnt, il.status,
                                             bl.keys, pair_capacity, rerender != 0,
                                             ctx && 2 * ctx->last_visible.load() > (long long)f->P, s));
    if ((rc = debug_sync(f, s, "emit"))) return rc;
    {
        const bool prof = ctx && ctx->profile;
        cudaEvent_t* pe = prof ? ctx->pev + 2 * 3 : nullptr;   // [start sort, end sort, start big, end big]
        gs_launch_tile_sort(G, ctx ? ctx->num_sms : g_gs_num_sms, il.tile_off, il.tile_cnt, il.status, il.big_list, bl.keys,
                            bl.list, pair_capacity, s, pe);
        if (prof) ctx->pev_used[3] = ctx->pev_used[4] = true;
    }
    if ((rc = debug_sync(f, s, "tile_sort"))) return rc;
    GS_TIMED(ctx, 5, s, gs_launch_blend_fwd(v, il.tile_off, bl.list, gl.rec, il.status, pair_capacity, il.final_T,
                                                il.n_contrib, out_color, out_depth, s));
    if ((rc = debug_sync(f, s, "blend_fwd"))) return rc;
    return GS_OK;
}

int gs_forward_views(GsContext* ctx, const GsFrame* frames, int32_t n_views, const GsViewScratch* scratch,
                     int32_t n_streams, GsViewResult* results, gs_stream_t stream) {
    if (!ctx || !frames || !scratch || !results) return fail(GS_EINVAL, "NULL argument");
    if (n_views < 0 || n_views > GS_STATUS_SLOTS) return fail(GS_EINVAL, "n_views must be in [0, %d]", GS_STATUS_SLOTS);
    if (n_streams < 1 || n_streams > kMaxViewStreams) return fail(GS_EINVAL, "n_streams must be in [1, %d]", kMaxViewStreams);
    if (n_views == 0) return GS_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int prev = 0;
    GS_CUDA(cudaGetDevice(&prev));
    GS_CUDA(cudaSetDevice(ctx->device));
    if (!ctx->vstreams_ready) {
        GS_CUDA(cudaEventCreateWithFlags(&ctx->vfork, cudaEventDisableTiming));
        for (int i = 0; i < kMaxViewStreams; i++) {
            GS_CUDA(cudaStreamCreateWithFlags(&ctx->vstreams[i], cudaStreamNonBlocking));
            GS_CUDA(cudaEventCreateWithFlags(&ctx->vjoin[i], cudaEventDisableTiming));
        }
        ctx->vstreams_ready = true;
    }
    const int ns = n_streams < n_views ? n_streams : n_views;
    GS_CUDA(cudaEventRecord(ctx->vfork, s));                       // fork: the views start after the caller's work
    for (int i = 0; i < ns; i++) GS_CUDA(cudaStreamWaitEvent(ctx->vstreams[i], ctx->vfork, 0));
    int32_t tickets[GS_STATUS_SLOTS];
    int rc = GS_OK;
    for (int k = 0; k < n_views && rc == GS_OK; k++) {
        const GsViewScratch& sc = scratch[k % ns];
        GsViewResult& r = results[k];
        cudaStream_t vs = ctx->vstreams[k % ns];
        int32_t* radii = r.radii ? r.radii : sc.radii;
        r.status = GS_OK;
        rc = gs_forward_preprocess(ctx, &frames[k], sc.geom_buffer, sc.image_buffer, radii, vs, &tickets[k]);
        if (rc == GS_OK)       // speculative: the device-side capacity guard skips the render if the buffer is too small
            rc = gs_forward_render(ctx, &frames[k], radii, sc.geom_buffer, sc.binning_buffer, sc.pair_capacity,
                                   sc.image_buffer, r.out_color, r.out_depth, 0, vs);
    }
    for (int i = 0; i < ns; i++) {                                 // join, also on the error path
        cudaEventRecord(ctx->vjoin[i], ctx->vstreams[i]);
        cudaStreamWaitEvent(s, ctx->vjoin[i], 0);
    }
    cudaSetDevice(prev);
    if (rc != GS_OK) return rc;
    for (int k = 0; k < n_views; k++) {                            // only now does the host wait, once per view
        const int rc2 = gs_forward_counts(ctx, tickets[k], &results[k].counts);
        if (rc2 != GS_OK) return rc2;
        if (results[k].counts.num_pairs > scratch[k % ns].pair_capacity) { results[k].status = GS_ECAPACITY; rc = GS_ECAPACITY; }
    }
    if (rc == GS_ECAPACITY) fail(GS_ECAPACITY, "at least one view needs a larger binning buffer (see results[].status)");
    return rc;
}

size_t gs_backward_scratch_bytes(int64_t num_visible) {
    return gs_align_up((size_t)(num_visible > 0 ? num_visible : 1) * GS_GOUT_FLOATS * sizeof(float), 256);
}

static GsGradPtrs grad_ptrs(const GsFrame* f, const GsGrads* grads) {
    GsGradPtrs g;
    g.dmeans3D = grads->dL_dmeans3D; g.dmeans2D = grads->dL_dmeans2D; g.dsh = f->shs ? grads->dL_dsh : nullptr;
    g.dcolors = grads->dL_dcolors; g.dopacity = grads->dL_dopacity;
    g.dscales = grads->dL_dscales; g.drots = grads->dL_drotations; g.dcov3D = grads->dL_dcov3D;
    return g;
}

static int ensure_aux(GsContext* ctx) {
    if (ctx->aux_ready) return GS_OK;
    int prev = 0;
    GS_CUDA(cudaGetDevice(&prev));
    GS_CUDA(cudaSetDevice(ctx->device));
    // highest priority: the block scheduler hands freed SM resources to the side stream's small CTAs first; at equal
    // priority they would wait until the tile pass (8 160 CTAs, launched into the caller's stream at the same moment)
    // has nothing left to dispatch, i.e. run AFTER it
    int pr_least = 0, pr_greatest = 0;
    GS_CUDA(cudaDeviceGetStreamPriorityRange(&pr_least, &pr_greatest));
    GS_CUDA(cudaStreamCreateWithPriority(&ctx->aux, cudaStreamNonBlocking, pr_greatest));
    GS_CUDA(cudaEventCreateWithFlags(&ctx->aux_fork, cudaEventDisableTiming));
    GS_CUDA(cudaEventCreateWithFlags(&ctx->aux_join, cudaEventDisableTiming));
    GS_CUDA(cudaSetDevice(prev));
    ctx->aux_ready = true;
    return GS_OK;
}

// Which kernels write the per-Gaussian gradients of one backward call, decided once from its inputs.
enum class GradWriter { none, tma, generic };
struct GradPlan {
    bool fill;          // k_fill_zero zeroes the outputs on ctx->aux beside the tile pass; k_grad_vis scatters final rows
    bool dense_ok;      // k_grad_dense covers the input mode: in its regime (decided on the device) the others exit
    bool dense;         // ... and is launched: the scratch bound does not prove the sparse regime
    GradWriter writer;  // the writer after k_grad_vis
    bool peer;          // rows are reduced into every rank's bucket (k_grad_reduce_peers); only dL_dmeans2D is local
    bool peer_begin;    // the peer route's "every bucket is cleared" barrier waits on ctx->aux beside the tile pass
};

// `nvis_bound`: compact rows the gradient scratch holds.  The TMA paths (k_fill_zero + scatter, k_grad_write_tma) need
// the six outputs of the reference's own input mode (16 stored SH coefficients) and nothing else, 16-byte aligned;
// k_grad_dense also needs scales + rotations and 16-byte aligned means / scales for its bulk copies (gsraster.h); the
// fill also needs P a multiple of 4 and a context for its side stream.
static GradPlan grad_plan(const GsContext* ctx, const GsFrame* f, const GsGrads* grads, const GsGradPtrs& g,
                          long long nvis_bound) {
    auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    const bool tma_ok = f->shs && f->M == 16 && g.dsh && g.dmeans3D && g.dmeans2D && g.dscales && g.dopacity && g.drots &&
                        !g.dcolors && !g.dcov3D && al16(g.dsh) && al16(g.dmeans3D) && al16(g.dmeans2D) &&
                        al16(g.dscales) && al16(g.dopacity) && al16(g.drots);
    const bool sr = !f->cov3D_precomp && f->scales && f->rotations;
    GradPlan p;
    p.peer = grads->peer_world > 0;
    p.peer_begin = ctx && p.peer && grads->peer_signals && grads->peer_epoch_begin;
    p.fill = ctx && f->P > 0 && !p.peer && !(f->P & 3) && sr && tma_ok;
    p.dense_ok = !p.peer && tma_ok && sr && al16(f->means3D) && al16(f->scales);
    p.dense = p.dense_ok && 2 * nvis_bound > (long long)f->P;
    p.writer = (p.peer || p.fill) ? GradWriter::none : tma_ok ? GradWriter::tma : GradWriter::generic;
    return p;
}

// The backward shared by gs_backward and gs_backward_deterministic once their own arguments are checked.  Tile pass:
// k_blend_bwd, or (`det` non-NULL) k_tile_partials + the fixed-order reduce.  Beside it on the context's side stream:
// the zero-fill of the outputs or the peer route's begin barrier.  Then the per-Gaussian writers of the plan, into the
// caller's tensors (or every rank's bucket).  `grad_scratch_bytes`: the compact-row part of the scratch.
static int backward_body(GsContext* ctx, const GsFrame* f, const int32_t* radii, const void* geom_buffer,
                         const void* binning_buffer, int64_t pair_capacity, const void* image_buffer, void* grad_scratch,
                         size_t grad_scratch_bytes, const float* dL_dout_color, const GsGrads* grads,
                         const GsDetLayout* det, gs_stream_t stream) {
    int rc = check_frame(f);
    if (rc) return rc;
    if (f->P > 0) {
        if (!geom_buffer || !binning_buffer || !image_buffer || !dL_dout_color)
            return fail(GS_EINVAL, "scratch / dL_dout_color is NULL");
        if (!radii || !grad_scratch) return fail(GS_EINVAL, "radii / scratch is NULL");
        if (grads->peer_world > GS_MAX_PEERS || (grads->peer_world > 0 && !grads->peer_buckets))
            return fail(GS_EINVAL, "bad peer arguments");
    }
    cudaStream_t s = (cudaStream_t)stream;
    const GsGradPtrs g = grad_ptrs(f, grads);
    const GradPlan plan = grad_plan(ctx, f, grads, g, (long long)(grad_scratch_bytes / (GS_GOUT_FLOATS * sizeof(float))));
    GsImageLayout il = gs_image_layout(const_cast<void*>(image_buffer), f->W, f->H);
    if (plan.fill || plan.peer_begin) {
        if ((rc = ensure_aux(ctx))) return rc;
        GS_CUDA(cudaEventRecord(ctx->aux_fork, s));        // the outputs were allocated in `stream` order before this call
        GS_CUDA(cudaStreamWaitEvent(ctx->aux, ctx->aux_fork, 0));
        // the tile pass is issue bound and leaves the memory system idle; in the dense regime the fill exits on the device
        if (plan.fill) GS_TIMED(ctx, 11, ctx->aux, gs_launch_fill_zero(f->P, ctx->num_sms, g, il.status, plan.dense_ok, ctx->aux));
        else gs_launch_peer_barrier((uint32_t* const*)grads->peer_signals, grads->peer_world, grads->peer_rank, 0,
                                    grads->peer_epoch_begin, ctx->aux);
        GS_CUDA(cudaEventRecord(ctx->aux_join, ctx->aux));
    }
    if (f->P == 0) return GS_OK;
    const GsView v = make_view(f);
    const int nsm = ctx ? ctx->num_sms : g_gs_num_sms;
    GsGeomLayout gl = gs_geom_layout(const_cast<void*>(geom_buffer), f->P);
    GsBinLayout bl = gs_bin_layout(const_cast<void*>(binning_buffer), pair_capacity > 0 ? pair_capacity : 1);
    if (!det) {
        GS_TIMED(ctx, 6, s, gs_launch_blend_bwd(v, il.tile_off, bl.list, gl.rec, il.final_T, il.n_contrib, dL_dout_color,
                                                gl.acc, il.status, pair_capacity, s));
        if ((rc = debug_sync(f, s, "blend_bwd"))) return rc;
    } else {
        gs_launch_tile_partials(v, il.tile_off, bl.list, gl.rec, il.final_T, il.n_contrib, dL_dout_color, det->part_a,
                                det->part_b, il.status, pair_capacity, s);
        if ((rc = debug_sync(f, s, "tile_partials"))) return rc;
        gs_launch_det_reduce(*det, nsm, bl.list, gl.vis_list, gl.acc, il.status, pair_capacity, s);
        if ((rc = debug_sync(f, s, "det_reduce"))) return rc;
    }

    float* gout = (float*)grad_scratch;
    if (plan.fill) GS_CUDA(cudaStreamWaitEvent(s, ctx->aux_join, 0));
    GS_TIMED(ctx, 7, s, gs_launch_grad_vis(v, nsm, f->means3D, f->shs, f->cov3D_precomp ? nullptr : f->scales,
                                           f->cov3D_precomp ? nullptr : f->rotations, f->cov3D_precomp, gl.rec, gl.acc,
                                           gl.vis_list, il.status, gout, plan.dense_ok, plan.fill, g, s));
    if ((rc = debug_sync(f, s, "grad_vis"))) return rc;
    if (plan.peer) {
        // nobody adds into a bucket before every rank has cleared its own
        if (plan.peer_begin) GS_CUDA(cudaStreamWaitEvent(s, ctx->aux_join, 0));
        GS_TIMED(ctx, 9, s, gs_launch_grad_reduce_peers(f->P, v.M, radii, gl.acc, gout, grads->dL_dmeans2D,
                                                        (float* const*)grads->peer_buckets, grads->peer_world,
                                                        (float*)grads->peer_multicast, (const long long*)grads->peer_seg_off, s));
        // the step's result is complete on this rank when every rank's adds have landed
        if (ctx && grads->peer_signals && grads->peer_epoch_end)
            gs_launch_peer_barrier((uint32_t* const*)grads->peer_signals, grads->peer_world, grads->peer_rank, 1,
                                   grads->peer_epoch_end, s);
        return debug_sync(f, s, "grad_reduce_peers");
    }
    if (plan.writer != GradWriter::none) {
        GS_TIMED(ctx, 9, s, gs_launch_grad_write(f->P, v.M, radii, gl.acc, gout, g, il.status, plan.dense_ok,
                                                 plan.writer == GradWriter::tma, s));
        if ((rc = debug_sync(f, s, "grad_write"))) return rc;
    }
    if (plan.dense) {
        GS_TIMED(ctx, 10, s, gs_launch_grad_dense(v, nsm, f->means3D, f->shs, f->scales, f->rotations, radii, gl.acc,
                                                  il.status, g, s));
        if ((rc = debug_sync(f, s, "grad_dense"))) return rc;
    }
    // outputs the fused kernel does not produce in this input mode are defined as zeros (reference: torch::zeros)
    const size_t Ps = (size_t)f->P;
    if (!f->shs && grads->dL_dsh && f->M > 0) GS_CUDA(cudaMemsetAsync(grads->dL_dsh, 0, Ps * f->M * 3 * sizeof(float), s));
    return GS_OK;
}

int gs_backward(GsContext* ctx, const GsFrame* f, const int32_t* radii, const void* geom_buffer,
                const void* binning_buffer, int64_t pair_capacity, const void* image_buffer, void* grad_scratch,
                size_t grad_scratch_bytes, const float* dL_dout_color, const float* dL_dout_depth,
                const GsGrads* grads, gs_stream_t stream) {
    (void)dL_dout_depth;                                 // depth gradient disabled in the reference
    if (!grads) return fail(GS_EINVAL, "grads is NULL");
    return backward_body(ctx, f, radii, geom_buffer, binning_buffer, pair_capacity, image_buffer, grad_scratch,
                         grad_scratch_bytes, dL_dout_color, grads, nullptr, stream);
}

// Bytes of the deterministic backward's scratch for `num_visible` compact slots and `pair_capacity` pairs: the default
// gradient scratch first, then the partials and the Gaussian-major pair index (GsDetLayout).
static size_t det_scratch_bytes(long long V, long long C) {
    return gs_backward_scratch_bytes(V) + gs_det_layout(nullptr, V, C).bytes;
}

size_t gs_backward_deterministic_scratch_bytes(int64_t num_visible, int64_t pair_capacity) {
    return det_scratch_bytes(num_visible > 0 ? num_visible : 1, pair_capacity > 0 ? pair_capacity : 1);
}

// The deterministic tile pass stores per-(tile, splat) partials by list position and sums them per Gaussian in
// ascending list position into the accumulators (gs_det_bwd.cu): the same accumulator contents as k_blend_bwd up to
// the order of the float additions, which is fixed here.
int gs_backward_deterministic(GsContext* ctx, const GsFrame* f, const int32_t* radii, const void* geom_buffer,
                              const void* binning_buffer, int64_t pair_capacity, const void* image_buffer,
                              void* grad_scratch, size_t grad_scratch_bytes, const float* dL_dout_color,
                              const float* dL_dout_depth, const GsGrads* grads, gs_stream_t stream) {
    (void)dL_dout_depth;                                 // depth gradient disabled in the reference
    if (!grads) return fail(GS_EINVAL, "grads is NULL");
    if (grads->peer_world > 0)
        return fail(GS_EINVAL, "gs_backward_deterministic does not support the peer reduce (peer_world > 0): "
                               "the cross-rank adds are not in a fixed order; use gs_backward");
    if (pair_capacity < 0) return fail(GS_EINVAL, "pair_capacity < 0");
    const long long C = pair_capacity > 0 ? pair_capacity : 1;
    // the number of compact slots the scratch was sized for: the largest V with det_scratch_bytes(V, C) <= the size given
    if (!grad_scratch || grad_scratch_bytes < det_scratch_bytes(1, C))
        return fail(GS_EINVAL, "grad_scratch must hold gs_backward_deterministic_scratch_bytes(num_visible, pair_capacity)"
                               " = at least %zu bytes", det_scratch_bytes(1, C));
    long long lo = 1, hi = (long long)(grad_scratch_bytes / (GS_GOUT_FLOATS * sizeof(float))) + 1;
    while (hi - lo > 1) {
        const long long mid = lo + (hi - lo) / 2;
        if (det_scratch_bytes(mid, C) <= grad_scratch_bytes) lo = mid; else hi = mid;
    }
    const long long V = lo;
    const size_t default_bytes = gs_backward_scratch_bytes(V);
    const GsDetLayout d = gs_det_layout((char*)grad_scratch + default_bytes, V, C);
    // the compact rows bound the visible count by the default part of the scratch only
    return backward_body(ctx, f, radii, geom_buffer, binning_buffer, pair_capacity, image_buffer, grad_scratch,
                         default_bytes, dL_dout_color, grads, &d, stream);
}

int gs_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    uint8_t* present, gs_stream_t stream) {
    (void)projmatrix;
    if (P < 0) return fail(GS_EINVAL, "P < 0");
    if (P == 0) return GS_OK;
    if (!means3D || !viewmatrix || !present) return fail(GS_EINVAL, "NULL argument");
    gs_launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "mark_visible launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_l1_loss_backward(GsContext* ctx, const float* color, const uint8_t* target_u8, int32_t H, int32_t W, float weight,
                        float* dL_dcolor, float* loss, gs_stream_t stream) {
    if (!color || !target_u8 || !dL_dcolor || !loss || H <= 0 || W <= 0) return fail(GS_EINVAL, "bad argument");
    gs_launch_l1_loss_grad(color, target_u8, H, W, weight, dL_dcolor, loss, ctx ? ctx->num_sms : g_gs_num_sms, (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "l1_loss launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_gaussian_adam_step(GsContext* ctx, const GsAdamGroup* groups, int32_t ngroups, double beta1, double beta2,
                          double eps, int32_t step, gs_stream_t stream) {
    (void)ctx;
    if (!groups || ngroups <= 0 || ngroups > 8 || step < 1) return fail(GS_EINVAL, "bad optimiser arguments");
    GsAdamArgs a;
    a.nseg = ngroups; a.om_beta1 = (float)(1.0 - beta1); a.beta2 = (float)beta2; a.om_beta2 = (float)(1.0 - beta2);
    a.eps = (float)eps;
    const double bc1 = 1.0 - pow(beta1, (double)step);
    a.bc2_sqrt = (float)sqrt(1.0 - pow(beta2, (double)step));
    for (int k = 0; k < ngroups; k++) {
        const GsAdamGroup& g = groups[k];
        if (!g.param || !g.grad || !g.exp_avg || !g.exp_avg_sq || g.rows < 0 || g.activation < 0 || g.activation > 3)
            return fail(GS_EINVAL, "optimiser group %d is malformed", k);
        if ((reinterpret_cast<uintptr_t>(g.param) | reinterpret_cast<uintptr_t>(g.exp_avg) |
             reinterpret_cast<uintptr_t>(g.exp_avg_sq)) & 15)
            return fail(GS_EINVAL, "optimiser group %d: param / moments must be 16-byte aligned", k);
        GsAdamSeg& s = a.seg[k];
        s.type = g.activation; s.row_w = g.activation == 3 ? 4 : g.row_width; s.g_row_w = g.grad_row_width;
        s.g_off = g.grad_offset; s.rows = g.rows; s.p = g.param; s.g = g.grad; s.m = g.exp_avg; s.v = g.exp_avg_sq;
        s.step_size = (float)(g.lr / bc1); s.blocks = 0;
        if (s.row_w <= 0 || s.g_row_w < s.row_w + s.g_off) return fail(GS_EINVAL, "optimiser group %d: bad row widths", k);
    }
    if (gs_launch_gaussian_adam(a, (cudaStream_t)stream) != 0) return fail(GS_EINVAL, "optimiser problem too large");
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "adam launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

static bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

// The status block of a guarded step's forward, or NULL (no guard).  -1: bad arguments.
static int guard_status(const void* image_buffer, int32_t W, int32_t H, int64_t pair_capacity, const GsDevStatus** out) {
    *out = nullptr;
    if (!image_buffer) return 0;
    if (W <= 0 || H <= 0 || pair_capacity < 0 || misaligned(image_buffer, 8)) return -1;
    *out = gs_image_layout(const_cast<void*>(image_buffer), W, H).status;
    return 0;
}

int gs_activate(GsContext* ctx, int32_t P, int32_t M, const float* features_dc, const float* features_rest,
                const float* opacity, const float* scaling, const float* rotation, float* shs, float* opacities,
                float* scales, float* rotations, gs_stream_t stream) {
    (void)ctx;
    if (P < 0 || M < 1 || M > 16) return fail(GS_EINVAL, "bad sizes P=%d M=%d", P, M);
    if (P == 0) return GS_OK;
    if (!features_dc || (M > 1 && !features_rest) || !opacity || !scaling || !rotation || !shs || !opacities || !scales ||
        !rotations)
        return fail(GS_EINVAL, "NULL argument");
    if (misaligned(rotation, 16) || misaligned(shs, 16) || misaligned(rotations, 16))
        return fail(GS_EINVAL, "rotation, shs and rotations must be 16-byte aligned");
    if (misaligned(features_dc, 4) || misaligned(features_rest, 4) || misaligned(opacity, 4) || misaligned(scaling, 4) ||
        misaligned(opacities, 4) || misaligned(scales, 4))
        return fail(GS_EINVAL, "features, opacity, scaling and their outputs must be 4-byte aligned");
    gs_launch_activate(P, M, features_dc, features_rest, opacity, scaling, rotation, shs, opacities, scales, rotations,
                       (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "activate launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

size_t gs_adam_sched_scratch_bytes(void) { return gs_align_up(sizeof(GsAdamSchedOut), 256); }

static bool betas_ok(double beta1, double beta2) { return beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0; }

int32_t gs_adam_bias_table_len(double beta1, double beta2) {
    if (!betas_ok(beta1, beta2)) return 0;
    for (int32_t s = 1; s < (1 << 24); s++)
        if (1.0 - pow(beta1, (double)s) == 1.0 && (float)sqrt(1.0 - pow(beta2, (double)s)) == 1.0f) return s + 1;
    return 0;
}

int gs_adam_bias_table(double beta1, double beta2, int32_t n, double* bc1, float* bc2_sqrt) {
    if (!betas_ok(beta1, beta2) || n < 2 || !bc1 || !bc2_sqrt) return fail(GS_EINVAL, "bad bias table arguments");
    for (int32_t s = 0; s < n; s++) {             // exactly gs_gaussian_adam_step's formation
        bc1[s] = 1.0 - pow(beta1, (double)s);
        bc2_sqrt[s] = (float)sqrt(1.0 - pow(beta2, (double)s));
    }
    return GS_OK;
}

int gs_gaussian_adam_sched_step(GsContext* ctx, const GsAdamSchedGroup* groups, int32_t ngroups, double beta1,
                                double beta2, double eps, const double* bias_bc1, const float* bias_bc2_sqrt,
                                int32_t bias_len, const int32_t* iteration, int32_t lr_table_len,
                                const void* image_buffer, int32_t W, int32_t H, int64_t pair_capacity, void* scratch,
                                size_t scratch_bytes, gs_stream_t stream) {
    (void)ctx;
    if (!groups || ngroups <= 0 || ngroups > 8 || !betas_ok(beta1, beta2))
        return fail(GS_EINVAL, "bad optimiser arguments");
    if (!bias_bc1 || !bias_bc2_sqrt || bias_len < 2 || misaligned(bias_bc1, 8) || misaligned(bias_bc2_sqrt, 4))
        return fail(GS_EINVAL, "bias-correction tables are NULL, misaligned or shorter than 2 entries");
    if (!scratch || misaligned(scratch, 16) || scratch_bytes < gs_adam_sched_scratch_bytes())
        return fail(GS_EINVAL, "scratch must hold gs_adam_sched_scratch_bytes() bytes, 16-byte aligned");
    GsAdamSched sc = {};
    if (guard_status(image_buffer, W, H, pair_capacity, &sc.status) != 0)
        return fail(GS_EINVAL, "guard: image buffer misaligned or bad W / H / pair_capacity");
    GsAdamArgs a;
    a.nseg = ngroups; a.om_beta1 = (float)(1.0 - beta1); a.beta2 = (float)beta2; a.om_beta2 = (float)(1.0 - beta2);
    a.eps = (float)eps; a.bc2_sqrt = 0.f;
    bool tables = false;
    for (int k = 0; k < ngroups; k++) {
        const GsAdamSchedGroup& g = groups[k];
        if (!g.param || !g.grad || !g.exp_avg || !g.exp_avg_sq || !g.step || g.rows < 0 || g.activation < 0 ||
            g.activation > 3)
            return fail(GS_EINVAL, "optimiser group %d is malformed", k);
        if (misaligned(g.param, 16) || misaligned(g.exp_avg, 16) || misaligned(g.exp_avg_sq, 16) || misaligned(g.grad, 4) ||
            misaligned(g.step, 4) || misaligned(g.lr_table, 8))
            return fail(GS_EINVAL, "optimiser group %d: param / moments must be 16-byte aligned, step 4, lr_table 8", k);
        GsAdamSeg& s = a.seg[k];
        s.type = g.activation; s.row_w = g.activation == 3 ? 4 : g.row_width; s.g_row_w = g.grad_row_width;
        s.g_off = g.grad_offset; s.rows = g.rows; s.p = g.param; s.g = g.grad; s.m = g.exp_avg; s.v = g.exp_avg_sq;
        s.step_size = 0.f; s.blocks = 0;
        if (s.row_w <= 0 || s.g_off < 0 || s.g_row_w < s.row_w + s.g_off)
            return fail(GS_EINVAL, "optimiser group %d: bad row widths", k);
        sc.step[k] = g.step; sc.lr_table[k] = g.lr_table; sc.lr[k] = g.lr;
        tables = tables || g.lr_table != nullptr;
    }
    if (tables && (!iteration || misaligned(iteration, 4) || lr_table_len < 1))
        return fail(GS_EINVAL, "a learning-rate table needs the device iteration and lr_table_len >= 1");
    sc.bias_bc1 = bias_bc1; sc.bias_bc2_sqrt = bias_bc2_sqrt; sc.bias_len = bias_len;
    sc.iteration = iteration; sc.lr_table_len = lr_table_len; sc.capacity = pair_capacity;
    sc.out = static_cast<GsAdamSchedOut*>(scratch);
    if (gs_launch_gaussian_adam_sched(a, sc, (cudaStream_t)stream) != 0) return fail(GS_EINVAL, "optimiser problem too large");
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "scheduled adam launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_densify_stats_guarded(GsContext* ctx, int32_t P, const int32_t* radii, const float* dL_dmeans2D,
                             float* xyz_gradient_accum, float* denom, float* max_radii2D, const void* image_buffer,
                             int32_t W, int32_t H, int64_t pair_capacity, gs_stream_t stream) {
    (void)ctx;
    if (P < 0 || (P > 0 && (!radii || !dL_dmeans2D || !xyz_gradient_accum || !denom || !max_radii2D)))
        return fail(GS_EINVAL, "bad argument");
    if (misaligned(radii, 4) || misaligned(dL_dmeans2D, 4) || misaligned(xyz_gradient_accum, 4) || misaligned(denom, 4) ||
        misaligned(max_radii2D, 4))
        return fail(GS_EINVAL, "radii, dL_dmeans2D and the accumulators must be 4-byte aligned");
    const GsDevStatus* status = nullptr;
    if (guard_status(image_buffer, W, H, pair_capacity, &status) != 0)
        return fail(GS_EINVAL, "guard: image buffer misaligned or bad W / H / pair_capacity");
    if (P == 0) return GS_OK;
    gs_launch_densify_stats_guarded(P, radii, dL_dmeans2D, xyz_gradient_accum, denom, max_radii2D, status, pair_capacity,
                                    (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "guarded densify stats launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_pack_frame(GsContext* ctx, int32_t H, int32_t W, const float* color, const float* depth, uint8_t* rgb8,
                  float* neg_depth, uint32_t* minmax_state, gs_stream_t stream) {
    (void)ctx;
    if (H < 0 || W < 0 || (H * (int64_t)W > 0 && (!color || !rgb8 || (depth && !neg_depth))))
        return fail(GS_EINVAL, "bad argument");
    if ((int64_t)H * W > 0x7fffffffLL / 4) return fail(GS_EINVAL, "image too large");
    gs_launch_pack_frame(H * W, color, depth, rgb8, neg_depth, minmax_state, (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "pack frame launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_minmax_read(GsContext* ctx, uint32_t* minmax_state, float* minmax2, gs_stream_t stream) {
    (void)ctx;
    if (!minmax_state || !minmax2) return fail(GS_EINVAL, "NULL argument");
    gs_launch_minmax_decode(minmax_state, minmax2, (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "minmax decode launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

size_t gs_colorize_scratch_bytes(int32_t F) { return F > 0 ? gs_colorize_scratch_bytes_impl(F) : 0; }

int gs_colorize_depth(GsContext* ctx, int32_t F, int32_t H, int32_t W, const float* value, float invalid_val,
                      const uint8_t* lut_rgba, uint32_t background_rgba, void* scratch, size_t scratch_bytes,
                      uint8_t* rgba, float* vminmax, gs_stream_t stream) {
    (void)ctx;
    if (F <= 0 || H <= 0 || W <= 0) return fail(GS_EINVAL, "bad sizes F=%d H=%d W=%d", F, H, W);
    if ((int64_t)H * W > 0x7fffffffLL) return fail(GS_EINVAL, "frame too large");
    if (!value || !lut_rgba || !scratch || !rgba) return fail(GS_EINVAL, "NULL argument");
    if ((reinterpret_cast<uintptr_t>(value) | reinterpret_cast<uintptr_t>(lut_rgba) | reinterpret_cast<uintptr_t>(rgba) |
         reinterpret_cast<uintptr_t>(vminmax)) & 3)
        return fail(GS_EINVAL, "value, lut_rgba, rgba and vminmax must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(scratch) & 15) return fail(GS_EINVAL, "scratch must be 16-byte aligned");
    const size_t need = gs_colorize_scratch_bytes(F);
    if (scratch_bytes < need) return fail(GS_EINVAL, "scratch too small: %zu < %zu bytes", scratch_bytes, need);
    const int rc = gs_launch_colorize(F, H, W, value, invalid_val, reinterpret_cast<const uint32_t*>(lut_rgba),
                                      background_rgba, scratch, reinterpret_cast<uint32_t*>(rgba), vminmax,
                                      (cudaStream_t)stream);
    cudaError_t e = rc != 0 ? (cudaError_t)rc : cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "colorize launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

size_t gs_knn_scratch_bytes(int32_t P) { return P > 0 ? gs_knn_scratch_bytes_impl(P) : 256; }

int gs_knn_mean_dist2(GsContext* ctx, int32_t P, const float* points, void* scratch, float* mean_dist2, gs_stream_t stream) {
    (void)ctx;
    if (P < 0 || (P > 0 && (!points || !scratch || !mean_dist2))) return fail(GS_EINVAL, "bad argument");
    const int rc = gs_launch_knn(P, points, scratch, mean_dist2, (cudaStream_t)stream);
    if (rc == -1) return fail(GS_EINVAL, "knn: radix-sort temporary storage exceeds the scratch allowance");
    cudaError_t e = cudaPeekAtLastError();
    if (rc != 0 || e != cudaSuccess) return fail(GS_ECUDA, "knn launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_densify_stats(GsContext* ctx, int32_t P, const int32_t* radii, const float* dL_dmeans2D, float* xyz_gradient_accum,
                     float* denom, float* max_radii2D, gs_stream_t stream) {
    (void)ctx;
    if (P < 0 || (P > 0 && (!radii || !dL_dmeans2D || !xyz_gradient_accum || !denom || !max_radii2D)))
        return fail(GS_EINVAL, "bad argument");
    gs_launch_densify_stats(P, radii, dL_dmeans2D, xyz_gradient_accum, denom, max_radii2D, (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "densify stats launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

size_t gs_photometric_scratch_bytes(int32_t H, int32_t W) { return 256 + (size_t)9 * H * W * sizeof(float); }

int gs_photometric_loss_backward(GsContext* ctx, const float* image, const float* gt, int32_t H, int32_t W,
                                 float lambda_dssim, void* scratch, float* dL_dimage, float* loss3, gs_stream_t stream) {
    (void)ctx;
    if (!image || !gt || !scratch || !loss3 || H <= 0 || W <= 0) return fail(GS_EINVAL, "bad argument");
    gs_launch_photometric(image, gt, H, W, lambda_dssim, scratch, dL_dimage, loss3, (cudaStream_t)stream);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return fail(GS_ECUDA, "photometric loss launch: %s", cudaGetErrorString(e));
    return GS_OK;
}

int gs_debug_export_binning(const GsFrame* f, const void* binning_buffer, int64_t pair_capacity,
                            const void* image_buffer, uint32_t* ranges, uint32_t* point_list, int64_t max_pairs,
                            gs_stream_t stream) {
    if (!f || !binning_buffer || !image_buffer) return fail(GS_EINVAL, "NULL argument");
    cudaStream_t s = (cudaStream_t)stream;
    GsImageLayout il = gs_image_layout(const_cast<void*>(image_buffer), f->W, f->H);
    GsBinLayout bl = gs_bin_layout(const_cast<void*>(binning_buffer), pair_capacity > 0 ? pair_capacity : 1);
    const int G = ((f->W + GS_TILE - 1) / GS_TILE) * ((f->H + GS_TILE - 1) / GS_TILE);
    if (ranges) GS_CUDA(cudaMemcpyAsync(ranges, il.tile_off, (size_t)(G + 1) * 4, cudaMemcpyDeviceToDevice, s));
    if (point_list && max_pairs > 0)
        GS_CUDA(cudaMemcpyAsync(point_list, bl.list, (size_t)max_pairs * 4, cudaMemcpyDeviceToDevice, s));
    return GS_OK;
}

int gs_debug_blend_rows_per_warp(GsContext* ctx, int32_t W, int32_t H) {
    if (!ctx || W <= 0 || H <= 0) return fail(GS_EINVAL, "bad argument");
    GsView v{};
    v.W = W; v.H = H;
    v.gx = (W + GS_TILE - 1) / GS_TILE; v.gy = (H + GS_TILE - 1) / GS_TILE;
    return gs_blend_use_strips(v) ? 4 : 8;
}

}  // extern "C"
