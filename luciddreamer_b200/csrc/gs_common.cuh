// Shared device-side definitions of the H100 rasterizer (sm_90a).
// Data layout in HBM (all opaque to the caller, sized by gs_*_bytes()):
//
//  geom buffer   rec[P]  : 3 x float4 per Gaussian, written only for visible ones
//                          q0 = (x_pix, y_pix, conic_a, conic_b)
//                          q1 = (conic_c, opacity, r, g)
//                          q2 = (b, depth, clamped-bits, cull threshold -ln(255 opacity) - slack)
//                acc[P]  : 3 x float4 gradient accumulator per Gaussian (zeroed for visible ones by the
//                          forward; consumed and re-zeroed by the backward)
//                          a0 = (dmean2D.x, dmean2D.y, dconic.a, dconic.b)
//                          a1 = (dconic.c, dopacity, dcolor.r, dcolor.g)
//                          a2 = (dcolor.b, SH clamp bits, 0, compact slot)
//  image buffer  final_T[N] f32 | n_contrib[N] u32 | tile_off[G+1] u32 | tile_cnt[G] u32 | status
//  binning       keys[C] u64 = (depth_bits << 32 | gaussian_idx)  |  list[C] u32 (per tile, depth sorted)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define GS_TILE 16           // reference config.h:15-17
#define GS_TILE_PIX 256
#define GS_NEAR 0.2f         // auxiliary.h:154

struct GsDevStatus {         // lives at the end of the image buffer
    unsigned long long num_rendered;   // sum of rect areas (reference semantics)
    unsigned long long num_pairs;      // pairs binned
    unsigned long long num_visible;
    unsigned int overflow;             // set by k_emit when num_pairs > capacity at render time
    unsigned int n_big;                // tiles queued for k_tile_sort_big
    unsigned int n_mid;                // tiles queued for k_tile_sort_mid
    unsigned int pad;                  // ticket counter of k_count_tiles (last CTA out scans the histogram)
};

struct GsImageLayout {
    float* final_T;
    uint32_t* n_contrib;
    uint32_t* tile_off;      // [G+1] exclusive offsets
    uint32_t* tile_cnt;      // [G]   histogram, then reused as emission cursors
    uint32_t* big_list;      // [G]   tiles whose bucket exceeds the warp-sort capacity
    GsDevStatus* status;
    size_t bytes;
};

__host__ __device__ inline size_t gs_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

__host__ inline GsImageLayout gs_image_layout(void* base, int W, int H) {
    GsImageLayout L;
    const size_t N = (size_t)W * H;
    const size_t G = (size_t)((W + GS_TILE - 1) / GS_TILE) * ((H + GS_TILE - 1) / GS_TILE);
    char* p = (char*)base;
    size_t off = 0;
    L.final_T = (float*)(p + off);      off = gs_align_up(off + N * 4, 256);
    L.n_contrib = (uint32_t*)(p + off); off = gs_align_up(off + N * 4, 256);
    L.tile_off = (uint32_t*)(p + off);  off = gs_align_up(off + (G + 1) * 4, 256);
    L.big_list = (uint32_t*)(p + off);  off = gs_align_up(off + G * 4, 256);
    L.tile_cnt = (uint32_t*)(p + off);  off = gs_align_up(off + G * 4, 256);
    L.status = (GsDevStatus*)(p + off); off = gs_align_up(off + sizeof(GsDevStatus), 256);
    L.bytes = off;
    return L;
}

struct GsGeomLayout {
    float4* rec;          // [P][3]
    float4* acc;          // [P][3]
    uint32_t* vis_list;   // [P] compact list of visible Gaussian indices (first num_visible entries valid)
    uint32_t* hitmask;    // [P] per compact slot: which tiles of a small rect the splat reaches (histogram -> emission)
    size_t bytes;
};
__host__ inline GsGeomLayout gs_geom_layout(void* base, int P) {
    GsGeomLayout L;
    char* p = (char*)base;
    size_t off = 0;
    L.rec = (float4*)(p + off); off = gs_align_up(off + (size_t)P * 48, 256);
    L.acc = (float4*)(p + off); off = gs_align_up(off + (size_t)P * 48, 256);
    L.vis_list = (uint32_t*)(p + off); off = gs_align_up(off + (size_t)P * 4, 256);
    L.hitmask = (uint32_t*)(p + off); off = gs_align_up(off + (size_t)P * 4, 256);
    L.bytes = off;
    return L;
}

#define GS_MAX_PEERS 16
#define GS_GOUT_FLOATS 44    // compact per-visible-Gaussian gradient row (gs_gauss_bwd.cu)

struct GsBinLayout {
    unsigned long long* keys;
    uint32_t* list;
    size_t bytes;
};
__host__ inline GsBinLayout gs_bin_layout(void* base, long long cap) {
    GsBinLayout L;
    char* p = (char*)base;
    size_t off = 0;
    L.keys = (unsigned long long*)(p + off); off = gs_align_up(off + (size_t)cap * 8, 256);
    L.list = (uint32_t*)(p + off);           off = gs_align_up(off + (size_t)cap * 4, 256);
    L.bytes = off;
    return L;
}

// Extra scratch of the deterministic backward (gs_det_bwd.cu), after the default gradient scratch: per pair of capacity
// the nine stored partials (36 B), the pair's compact slot and its position in the Gaussian-major index (4 B each); per
// compact slot a count / cursor, a segment offset and a queue entry (4 B each).
struct GsDetLayout {
    float4* part_a;       // [2C] partials (a0, a1) of pair r at 2r, 2r+1 (32-byte aligned records)
    float* part_b;        // [C]  partial a2.x of pair r
    uint32_t* pair_slot;  // [C]  compact slot of pair r's Gaussian
    uint32_t* idx;        // [C]  pair positions grouped by slot (segment of slot s: [seg[s], seg[s+1])), ascending
    uint32_t* qcount;     // [2]  queued segments: <= 256 pairs (front of `queue`), longer (back)
    uint32_t* cnt;        // [V]  pairs per slot (directly after qcount: one clear covers both)
    uint32_t* seg;        // [V+1]
    uint32_t* queue;      // [V]
    uint32_t* bsum;       // [ceil(V / 2048)] scan block sums
    long long nslots;     // V
    size_t bytes;
};
__host__ inline GsDetLayout gs_det_layout(void* base, long long V, long long C) {
    GsDetLayout L;
    char* p = (char*)base;
    size_t off = 0;
    L.part_a = (float4*)(p + off);      off = gs_align_up(off + (size_t)C * 32, 256);
    L.part_b = (float*)(p + off);       off = gs_align_up(off + (size_t)C * 4, 256);
    L.pair_slot = (uint32_t*)(p + off); off = gs_align_up(off + (size_t)C * 4, 256);
    L.idx = (uint32_t*)(p + off);       off = gs_align_up(off + (size_t)C * 4, 256);
    L.qcount = (uint32_t*)(p + off);
    L.cnt = L.qcount + 2;               off = gs_align_up(off + (size_t)(V + 2) * 4, 256);
    L.seg = (uint32_t*)(p + off);       off = gs_align_up(off + (size_t)(V + 1) * 4, 256);
    L.queue = (uint32_t*)(p + off);     off = gs_align_up(off + (size_t)V * 4, 256);
    L.bsum = (uint32_t*)(p + off);      off = gs_align_up(off + (size_t)((V + 2047) / 2048) * 4, 256);
    L.nslots = V;
    L.bytes = off;
    return L;
}

// Per-view constants, passed by value to the kernels.  The camera matrices stay where the reference API puts
// them (device memory: raster_settings.viewmatrix / projmatrix / campos / bg are CUDA tensors); each CTA stages
// them into shared memory once (gs_load_cam) -- the host never reads them back.
struct GsView {
    const float* vm;      // [16] device
    const float* pm;      // [16] device
    const float* campos;  // [3]  device
    const float* bg;      // [3]  device
    float tan_fovx, tan_fovy, focal_x, focal_y, scale_modifier;
    int W, H, gx, gy, P, D, M;
};
struct GsCam {
    float vm[16];
    float pm[16];
    float campos[3];
    float bg[3];
};
// all threads of the CTA must call; contains a __syncthreads()
__device__ __forceinline__ void gs_load_cam(const GsView& v, GsCam* s_cam) {
    const int t = threadIdx.x;
    float* d = reinterpret_cast<float*>(s_cam);
    if (t < 16) d[t] = __ldg(v.vm + t);
    else if (t < 32) d[t] = __ldg(v.pm + (t - 16));
    else if (t < 35) d[t] = __ldg(v.campos + (t - 32));
    else if (t < 38) d[t] = __ldg(v.bg + (t - 35));
    __syncthreads();
}

// ---- small math helpers, same expression order as the oracle / reference formulas

__device__ __forceinline__ float3 gs_xf4x3(const float3 p, const float* m) {  // auxiliary.h:58-66
    return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
                       m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                       m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]);
}
__device__ __forceinline__ float4 gs_xf4x4(const float3 p, const float* m) {  // auxiliary.h:68-77
    return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
                       m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                       m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14],
                       m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}
__device__ __forceinline__ float gs_ndc2pix(float v, int S) {                // auxiliary.h:41-44 (double)
    return ((v + 1.0) * S - 1.0) * 0.5;
}
// auxiliary.h:46-56; returns rect as (xmin, ymin, xmax, ymax) in tiles
__device__ __forceinline__ int4 gs_rect(float px, float py, int r, int gx, int gy) {
    int4 q;
    q.x = min(gx, max(0, (int)((px - r) / GS_TILE)));
    q.y = min(gy, max(0, (int)((py - r) / GS_TILE)));
    q.z = min(gx, max(0, (int)((px + r + GS_TILE - 1) / GS_TILE)));
    q.w = min(gy, max(0, (int)((py + r + GS_TILE - 1) / GS_TILE)));
    return q;
}

struct GsCov2D {
    float tx, ty, tz;      // clamped view-space mean
    float xmul, ymul;
    float A[2][3];         // (J . V3) rows 0,1
    float a, b, c;         // cov2D + 0.3 I
};

// forward.cu:74-113 / backward.cu:158-207: A = J.V3, cov = A Sigma A^T, +0.3 on the diagonal
__device__ __forceinline__ void gs_cov2d(const float3 mean, const GsView& v, const float* vm, const float* c6,
                                         GsCov2D& o) {
    float3 t = gs_xf4x3(mean, vm);
    const float limx = 1.3f * v.tan_fovx, limy = 1.3f * v.tan_fovy;
    const float txtz = t.x / t.z, tytz = t.y / t.z;
    t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
    t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
    o.xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    o.ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    o.tx = t.x; o.ty = t.y; o.tz = t.z;
    const float J00 = v.focal_x / t.z, J02 = -(v.focal_x * t.x) / (t.z * t.z);
    const float J11 = v.focal_y / t.z, J12 = -(v.focal_y * t.y) / (t.z * t.z);
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const float v0 = vm[0 + 4 * j], v1 = vm[1 + 4 * j], v2 = vm[2 + 4 * j];
        o.A[0][j] = v0 * J00 + v1 * 0.f + v2 * J02;
        o.A[1][j] = v0 * 0.f + v1 * J11 + v2 * J12;
    }
    const float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
    float B[2][3];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int k = 0; k < 3; k++) B[i][k] = o.A[i][0] * S[0][k] + o.A[i][1] * S[1][k] + o.A[i][2] * S[2][k];
    o.a = (B[0][0] * o.A[0][0] + B[0][1] * o.A[0][1] + B[0][2] * o.A[0][2]) + 0.3f;
    o.b = (B[0][0] * o.A[1][0] + B[0][1] * o.A[1][1] + B[0][2] * o.A[1][2]);
    o.c = (B[1][0] * o.A[1][0] + B[1][1] * o.A[1][1] + B[1][2] * o.A[1][2]) + 0.3f;
}

// Rotation matrix of the un-normalised quaternion (r,x,y,z); forward.cu:127-139
__device__ __forceinline__ void gs_quat_R(const float4 q, float R[3][3]) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z);       R[0][2] = 2.f * (x * z + r * y);
    R[1][0] = 2.f * (x * y + r * z);       R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
    R[2][0] = 2.f * (x * z - r * y);       R[2][1] = 2.f * (y * z + r * x);       R[2][2] = 1.f - 2.f * (x * x + y * y);
}
// forward.cu:118-152: Sigma = R S S R^T (upper triangle)
__device__ __forceinline__ void gs_cov3d(const float3 s, float mod, const float4 q, float* c6) {
    float R[3][3], M[3][3];
    gs_quat_R(q, R);
    const float sv[3] = {mod * s.x, mod * s.y, mod * s.z};
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) M[i][j] = sv[i] * R[j][i];
#define GS_SIG(a, b) (M[0][a] * M[0][b] + M[1][a] * M[1][b] + M[2][a] * M[2][b])
    c6[0] = GS_SIG(0, 0); c6[1] = GS_SIG(0, 1); c6[2] = GS_SIG(0, 2);
    c6[3] = GS_SIG(1, 1); c6[4] = GS_SIG(1, 2); c6[5] = GS_SIG(2, 2);
#undef GS_SIG
}

// SH constants (auxiliary.h:22-39)
#define GS_C0 0.28209479177387814f
#define GS_C1 0.4886025119029199f
#define GS_C2_0 1.0925484305920792f
#define GS_C2_1 -1.0925484305920792f
#define GS_C2_2 0.31539156525252005f
#define GS_C2_3 -1.0925484305920792f
#define GS_C2_4 0.5462742152960396f
#define GS_C3_0 -0.5900435899266435f
#define GS_C3_1 2.890611442640554f
#define GS_C3_2 -0.4570457994644658f
#define GS_C3_3 0.3731763325901154f
#define GS_C3_4 -0.4570457994644658f
#define GS_C3_5 1.445305721320277f
#define GS_C3_6 -0.5900435899266435f

// SH basis (forward.cu:30-59); entries beyond the active degree are 0
__device__ __forceinline__ void gs_sh_basis(int deg, float x, float y, float z, float* b) {
#pragma unroll
    for (int k = 0; k < 16; k++) b[k] = 0.f;
    b[0] = GS_C0;
    if (deg > 0) {
        b[1] = -GS_C1 * y; b[2] = GS_C1 * z; b[3] = -GS_C1 * x;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = GS_C2_0 * xy; b[5] = GS_C2_1 * yz; b[6] = GS_C2_2 * (2.f * zz - xx - yy);
            b[7] = GS_C2_3 * xz; b[8] = GS_C2_4 * (xx - yy);
            if (deg > 2) {
                b[9] = GS_C3_0 * y * (3.f * xx - yy);
                b[10] = GS_C3_1 * xy * z;
                b[11] = GS_C3_2 * y * (4.f * zz - xx - yy);
                b[12] = GS_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy);
                b[13] = GS_C3_4 * x * (4.f * zz - xx - yy);
                b[14] = GS_C3_5 * z * (xx - yy);
                b[15] = GS_C3_6 * x * (xx - 3.f * yy);
            }
        }
    }
}

#define GS_REC_V4 3          // float4s per splat record
#define GS_CULL_SLACK 0.01f  // in units of `power` (~1 % in alpha): keeps the culling tests conservative

// Can a splat reach alpha >= 1/255 at some pixel of the box [x0,x1] x [y0,y1] (pixel-centre coordinates)?
// power(d) = -0.5 (A dx^2 + C dy^2) - B dx dy is concave with maximum 0 at the mean (mx,my): its maximum over the
// box is 0 if the mean is inside, otherwise it lies on an edge facing the mean, and each facing edge is a 1-D
// concave maximisation (clamp the stationary point to the edge).  thr = -ln(255 * opacity) - GS_CULL_SLACK, so
// "max power >= thr" is a conservative superset of "some pixel has alpha >= 1/255".  NaNs answer true (keep).
__device__ __forceinline__ bool gs_box_hit(float mx, float my, float A, float B, float C, float thr, float x0,
                                           float y0, float x1, float y1) {
    // the edge maximisation below needs a concave power(): a conic that is not positive definite (fp32 cancellation
    // on huge anisotropic splats, a non-PSD cov3D_precomp) is never culled
    if (!(A > 0.f && C > 0.f && A * C - B * B > 0.f)) return true;
    const bool in_x = mx >= x0 && mx <= x1, in_y = my >= y0 && my <= y1;
    if (in_x && in_y) return !(thr > 0.f);
    float best = -3.0e38f;
    if (!in_x) {                                         // facing vertical edge
        const float ex = mx < x0 ? x0 : x1;
        const float dx = mx - ex;
        float py = my + B * dx / C;                      // stationary point along the edge
        py = fminf(y1, fmaxf(y0, py));
        const float dy = my - py;
        best = fmaxf(best, -0.5f * (A * dx * dx + C * dy * dy) - B * dx * dy);
    }
    if (!in_y) {                                         // facing horizontal edge
        const float ey = my < y0 ? y0 : y1;
        const float dy = my - ey;
        float px = mx + B * dy / A;
        px = fminf(x1, fmaxf(x0, px));
        const float dx = mx - px;
        best = fmaxf(best, -0.5f * (A * dx * dx + C * dy * dy) - B * dx * dy);
    }
    return !(best < thr);
}

// Zeroes `words` 32-bit words with a KERNEL.  cudaMemsetAsync nodes may be served by a copy engine, where they queue
// behind whatever large host<->device transfer is in flight on another stream (a CUDA-graph step would stall behind
// the next step's 6 MB image upload); a kernel only depends on its own stream.
void gs_launch_clear_words(uint32_t* p, size_t words, cudaStream_t s);

// launchers (defined in the .cu files, used by gs_api.cu)
struct GsGradPtrs {
    float *dmeans3D, *dmeans2D, *dsh, *dcolors, *dopacity, *dscales, *drots, *dcov3D;
};
void gs_launch_project(const GsView& v, const float* means3D, const float* opacities, const float* scales,
                       const float* rotations, const float* cov3D_precomp, int* radii, float4* rec,
                       uint32_t* vis_list, GsDevStatus* status, bool dense_hint, cudaStream_t s);
void gs_launch_count_tiles(const GsView& v, int num_sms, const int* radii, const float4* rec, const uint32_t* vis_list,
                           uint32_t* hitmask, uint32_t* tile_cnt, GsDevStatus* status, uint32_t* tile_off,
                           GsDevStatus* host_slot, cudaStream_t s);
void gs_preprocess_init();
void gs_launch_tile_scan(int G, uint32_t* tile_cnt, uint32_t* tile_off, GsDevStatus* status,
                         GsDevStatus* host_slot, cudaStream_t s);
void gs_launch_shade_emit(const GsView& v, int num_sms, const float* means3D, const float* shs,
                          const float* colors_precomp, const int* radii, float4* rec, float4* acc,
                          const uint32_t* vis_list, const uint32_t* hitmask, const uint32_t* tile_off, uint32_t* tile_cur,
                          GsDevStatus* status, unsigned long long* keys, long long capacity, bool shaded, bool dense_hint,
                          cudaStream_t s);
void gs_tile_sort_init();
void gs_launch_tile_sort(int G, int num_sms, const uint32_t* tile_off, uint32_t* tile_cur, GsDevStatus* status,
                         uint32_t* big_list, unsigned long long* keys, uint32_t* list, long long capacity,
                         cudaStream_t s, cudaEvent_t* prof);
void gs_launch_blend_fwd(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                         const GsDevStatus* status, long long capacity, float* final_T, uint32_t* n_contrib,
                         float* out_color, float* out_depth, cudaStream_t s);
void gs_launch_blend_bwd(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                         const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, float4* acc,
                         const GsDevStatus* status, long long capacity, cudaStream_t s);
void gs_launch_tile_partials(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                             const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, float4* part_a,
                             float* part_b, const GsDevStatus* status, long long capacity, cudaStream_t s);
bool gs_blend_use_strips(const GsView& v);
void gs_det_bwd_init();
void gs_launch_det_reduce(const GsDetLayout& d, int num_sms, const uint32_t* list, const uint32_t* vis_list, float4* acc,
                          const GsDevStatus* status, long long capacity, cudaStream_t s);
extern int g_gs_num_sms;
void gs_launch_grad_vis(const GsView& v, int num_sms, const float* means3D, const float* shs, const float* scales,
                        const float* rotations, const float* cov3D_precomp, const float4* rec, float4* acc,
                        const uint32_t* vis_list, const GsDevStatus* status, float* gout, bool dense_elsewhere,
                        bool scatter, GsGradPtrs g, cudaStream_t s);
void gs_launch_fill_zero(int P, int num_sms, const GsGradPtrs& g, const GsDevStatus* status, bool dense_elsewhere,
                         cudaStream_t s);
void gs_launch_grad_dense(const GsView& v, int num_sms, const float* means3D, const float* shs, const float* scales,
                          const float* rotations, const int* radii, float4* acc, const GsDevStatus* status, GsGradPtrs g,
                          cudaStream_t s);
void gs_grad_write_init();
void gs_launch_grad_write(int P, int M, const int* radii, const float4* acc, const float* gout, GsGradPtrs g,
                          const GsDevStatus* status, bool dense_elsewhere, bool tma, cudaStream_t s);
void gs_launch_grad_reduce_peers(int P, int M, const int* radii, const float4* acc, const float* gout, float* dmeans2D,
                                 float* const* peers, int world, float* mc, const long long* seg_off,
                                 cudaStream_t s);
void gs_launch_peer_barrier(uint32_t* const* signals, int world, int rank, int channel, uint32_t epoch, cudaStream_t s);
void gs_launch_l1_loss_grad(const float* color, const uint8_t* target, int H, int W, float weight, float* dL_dcolor,
                            float* loss, int num_sms, cudaStream_t s);
void gs_launch_photometric(const float* img, const float* gt, int H, int W, float lambda_dssim, void* scratch,
                           float* dL_dimg, float* loss3, cudaStream_t s);
struct GsAdamSeg {
    int type;            // 0 identity, 1 sigmoid (opacity logit), 2 exp (log scale), 3 normalised quaternion rows
    int row_w;           // parameter row width (ignored for type 3: 4)
    int g_row_w, g_off;  // the gradient of parameter (row, c) sits at g[row * g_row_w + g_off + c]
    long long rows;
    float* p; const float* g; float* m; float* v;
    float step_size;     // lr / (1 - beta1^step)
    int blocks;
};
struct GsAdamArgs {
    GsAdamSeg seg[8];
    int nseg;
    float om_beta1, beta2, om_beta2, eps, bc2_sqrt;
};
int gs_launch_gaussian_adam(GsAdamArgs a, cudaStream_t s);
struct GsAdamSchedOut {      // per-step scalars k_adam_sched_prep hands to k_gaussian_adam_sched (device scratch)
    float step_size[8];
    float bc2_sqrt[8];
    int skip;                // the guarded frame overflowed: nothing is updated
};
struct GsAdamSched {         // where the scheduled Adam reads its scalars (all device pointers)
    float* step[8];                  // per-group step counter (float32, like torch's state["step"])
    const double* lr_table[8];       // per-iteration learning rate, or NULL: lr[g]
    double lr[8];
    const double* bias_bc1;          // [bias_len] 1 - beta1^s
    const float* bias_bc2_sqrt;      // [bias_len] sqrt(1 - beta2^s)
    int bias_len;
    int lr_table_len;
    const int* iteration;            // index into the lr tables
    const GsDevStatus* status;       // guard: the forward's status block, or NULL
    long long capacity;
    GsAdamSchedOut* out;
};
int gs_launch_gaussian_adam_sched(GsAdamArgs a, const GsAdamSched& sc, cudaStream_t s);
void gs_launch_activate(int P, int M, const float* f_dc, const float* f_rest, const float* opacity, const float* scaling,
                        const float* rotation, float* shs, float* opac_out, float* scale_out, float* rot_out,
                        cudaStream_t s);
void gs_launch_densify_stats_guarded(int P, const int* radii, const float* dm2, float* accum, float* denom,
                                     float* max_radii, const GsDevStatus* status, long long capacity, cudaStream_t s);
void gs_launch_pack_frame(int N, const float* color, const float* depth, uint8_t* rgb8, float* depth_out, unsigned* minmax,
                          cudaStream_t s);
void gs_launch_minmax_decode(unsigned* mm, float* out2, cudaStream_t s);
size_t gs_colorize_scratch_bytes_impl(int F);
int gs_launch_colorize(int F, int H, int W, const float* value, float invalid_val, const uint32_t* lut, uint32_t bg,
                       void* scratch, uint32_t* rgba, float* vminmax, cudaStream_t s);
size_t gs_knn_scratch_bytes_impl(int P);
int gs_launch_knn(int P, const float* points, void* scratch, float* out, cudaStream_t s);
void gs_launch_densify_stats(int P, const int* radii, const float* dm2, float* accum, float* denom, float* max_radii,
                             cudaStream_t s);
void gs_launch_mark_visible(int P, const float* means3D, const float* vm, uint8_t* present, cudaStream_t s);
