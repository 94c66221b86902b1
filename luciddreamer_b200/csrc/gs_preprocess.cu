// Per-Gaussian forward passes, tile histogram scan and (tile, Gaussian) pair emission for sm_90a.
//
// Replaces (RAST = reference rasterizer):
//   k_project      the geometric half of preprocessCUDA (RAST/cuda_rasterizer/forward.cu:155-232,249-255) +
//                  in_frustum (auxiliary.h:139-164): streaming pass over all P Gaussians, one thread each; visible
//                  ones are appended to a compact list (warp-aggregated atomic) so that every later per-Gaussian
//                  kernel runs densely over P_vis instead of divergently over P
//   k_count_tiles  the tile histogram over the compact list that replaces tiles_touched / InclusiveSum
//   k_tile_scan    cub::DeviceScan::InclusiveSum over P Gaussians + blocking D2H of num_rendered
//                  (rasterizer_impl.cu:278-282): here a scan over the G tiles only, totals mirrored to pinned
//                  host memory so the host never blocks the stream
//   k_shade_emit   the colour half (computeColorFromSH, forward.cu:20-71,236-246) on the compact list, 128-bit
//                  SH loads all in flight at once, + duplicateWithKeys (rasterizer_impl.cu:70-111): pairs go
//                  straight into their tile's bucket (per-tile cursors), keyed by (depth bits, Gaussian index).
//                  Runs AFTER the scan, i.e. after the point the host waits for, so shading overlaps the host
//   k_mark_visible checkFrustum (rasterizer_impl.cu:54-66)
// Histogram and emission spread the (Gaussian, tile) candidates of a CTA's 256 Gaussians evenly over its threads
// (block scan of the rect areas + binary search), so a splat covering thousands of tiles costs the same per thread
// as one covering four.

#include "gs_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kChunkMax = 256;        // Gaussians per CTA round in the vis-list kernels: 256 when many are visible (every
constexpr int kChunkMin = 64;         // thread owns one), 64 when only a few 10^4 are (small chunks keep all SMs busy; the
                                      // candidate walk uses all threads either way).  Chosen on the device from num_visible.
constexpr int kFoldK = 16;           // tiles per thread when the last CTA of k_count_tiles scans the histogram (two rounds at 1080p)
constexpr int kBitRect = 32;          // rects of up to 32 tiles: the histogram pass hands its hit decisions to the emission
                                      // pass as a bit mask (one word per visible Gaussian), so the exact test runs once

__device__ __forceinline__ int vis_chunk(uint32_t nvis) {
    return nvis >= (uint32_t)gridDim.x * (uint32_t)kChunkMax ? kChunkMax : kChunkMin;
}

// Exact tile culling (parity-safe, SURVEY.md Appendix B.4): a (tile, splat) pair is binned only if the splat can
// reach alpha >= 1/255 somewhere in the tile (gs_box_hit).  Pairs that are dropped are skipped by every pixel of
// the tile in the reference too (forward.cu:336-346), so no output changes.
// __noinline__: the histogram pass (k_count_tiles) and the emission pass (k_shade_emit) must take bit-identical
// decisions, so both call the same machine code on the same stored floats.
__device__ __noinline__ bool gs_tile_hit(float mx, float my, float A, float B, float C, float thr, int tx, int ty) {
    const float x0 = (float)(tx * GS_TILE), y0 = (float)(ty * GS_TILE);
    return gs_box_hit(mx, my, A, B, C, thr, x0, y0, x0 + (float)(GS_TILE - 1), y0 + (float)(GS_TILE - 1));
}

struct CandShared {                   // per-CTA candidate table (one entry per Gaussian of the chunk)
    float mx[kChunkMax], my[kChunkMax], A[kChunkMax], B[kChunkMax], C[kChunkMax], thr[kChunkMax];
    int rx[kChunkMax], ry[kChunkMax], rw[kChunkMax];
    uint32_t p0[kChunkMax], p1[kChunkMax];
    uint32_t bits[kChunkMax];         // hit bits of rects with <= kBitRect tiles (bit r = tile r of the rect, row-major)
    uint32_t cum[kChunkMax + 1];
    uint32_t warp_tot[kChunkMax / 32];
};

// Exclusive scan of the chunk's `area`s (threads 0..CH-1 hold one each) into s.cum[0..CH]; returns the total.
// All threads of the CTA must call.
__device__ __forceinline__ uint32_t cta_scan_areas(CandShared& s, uint32_t area, const int CH) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint32_t x = area;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s.warp_tot[wid] = x;                 // threads >= CH carry area 0
    __syncthreads();
    uint32_t wbase = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; w++) { const uint32_t t = s.warp_tot[w]; if (w < wid) wbase += t; total += t; }
    if (tid < CH) s.cum[tid] = wbase + x - area;
    if (tid == 0) s.cum[CH] = total;
    __syncthreads();
    return total;
}

// Visits every (Gaussian, tile) candidate of the chunk: f(valid, c, r, tx, ty) with c the chunk-local Gaussian, r the
// index of the tile inside its rect (row-major).  The candidates are spread evenly over the threads of the CTA; every
// thread runs the same number of rounds (lanes without a candidate in the last round get valid = false), so f may
// use warp-wide primitives.
template <typename F>
__device__ __forceinline__ void cta_for_each_candidate(const CandShared& s, uint32_t total, const int CH, F f) {
    if (total == 0) return;
    uint32_t q = threadIdx.x;
    int c = 0;
    for (uint32_t base = 0; base < total; base += kThreads, q += kThreads) {
        const bool valid = q < total;
        int r = 0, tx = 0, ty = 0;
        if (valid) {
            // largest c with cum[c] <= q.  Consecutive rounds are kThreads candidates apart: a step or two when the rects
            // are large, ~100 Gaussians when they are small -- a few linear steps, then a binary search in [c, CH)
            for (int k = 0; k < 3 && s.cum[c + 1] <= q; k++) c++;
            if (s.cum[c + 1] <= q) {
                int lo = c, hi = CH;
                while (hi - lo > 1) {
                    const int mid = (lo + hi) >> 1;
                    if (s.cum[mid] <= q) lo = mid; else hi = mid;
                }
                c = lo;
            }
            r = (int)(q - s.cum[c]);
            const int w = s.rw[c];
            const int yy = r / w, xx = r - yy * w;
            tx = s.rx[c] + xx; ty = s.ry[c] + yy;
        }
        f(valid, c, r, tx, ty);
    }
}

// Lanes of a warp that hit the SAME tile share one atomic: returns the lane's rank among them and, in `count`, how many
// they are; `leader` is true for the lane that issues the atomic.  Gaussians that are neighbours in memory are usually
// neighbours on screen (LucidDreamer's point clouds are in raster order, luciddreamer.py:363-372), so a warp's 32
// candidates mostly fall into one or two tiles.
__device__ __forceinline__ int tile_peers(const bool hit, const uint32_t tile, int& count, bool& leader, unsigned& peers) {
    const int lane = threadIdx.x & 31;
    peers = __match_any_sync(0xffffffffu, hit ? tile : (0x80000000u | (uint32_t)lane));
    count = __popc(peers);
    leader = hit && lane == __ffs(peers) - 1;
    return __popc(peers & ((1u << lane) - 1u));
}

// The exact per-Gaussian geometry of preprocessCUDA (forward.cu:155-232,249-255) for Gaussian i.
struct Projected {
    bool vis;
    int radius;
    float4 q0, q1;
};
__device__ __forceinline__ Projected project_exact(const int i, const GsView& v, const GsCam& cam,
                                                   const float* __restrict__ means3D, const float* __restrict__ opacities,
                                                   const float* __restrict__ scales, const float* __restrict__ rotations,
                                                   const float* __restrict__ cov3D_precomp) {
    Projected o;
    o.vis = false; o.radius = 0;
    o.q0 = make_float4(0.f, 0.f, 0.f, 0.f); o.q1 = o.q0;
    const float3 p = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
    const float3 p_view = gs_xf4x3(p, cam.vm);
    if (p_view.z > GS_NEAR) {                           // only the near plane culls (auxiliary.h:154)
        const float4 p_hom = gs_xf4x4(p, cam.pm);
        const float p_w = 1.0f / (p_hom.w + 0.0000001f);
        const float ppx = p_hom.x * p_w, ppy = p_hom.y * p_w;
        float c6[6];
        if (cov3D_precomp) {
#pragma unroll
            for (int k = 0; k < 6; k++) c6[k] = cov3D_precomp[6 * i + k];
        } else {
            const float3 s = make_float3(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]);
            const float4 q = __ldg(reinterpret_cast<const float4*>(rotations) + i);
            gs_cov3d(s, v.scale_modifier, q, c6);
        }
        GsCov2D cc;
        gs_cov2d(p, v, cam.vm, c6, cc);
        const float det = cc.a * cc.c - cc.b * cc.b;
        if (det != 0.0f) {
            const float det_inv = 1.f / det;
            const float3 conic = make_float3(cc.c * det_inv, -cc.b * det_inv, cc.a * det_inv);
            const float mid = 0.5f * (cc.a + cc.c);
            const float lambda1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det));
            const float lambda2 = mid - sqrtf(fmaxf(0.1f, mid * mid - det));
            const float rad = ceilf(3.f * sqrtf(fmaxf(lambda1, lambda2)));
            const float px = gs_ndc2pix(ppx, v.W), py = gs_ndc2pix(ppy, v.H);
            const int4 rect = gs_rect(px, py, (int)rad, v.gx, v.gy);
            if ((rect.z - rect.x) * (rect.w - rect.y) != 0) {
                o.vis = true;
                o.radius = (int)rad;
                const float opac = opacities[i];
                // alpha >= 1/255  <=>  power >= -ln(255 * opacity); slack keeps the test conservative
                const float thr = -logf(255.0f * opac) - GS_CULL_SLACK;
                o.q0 = make_float4(px, py, conic.x, conic.y);
                o.q1 = make_float4(conic.z, opac, p_view.z, thr);        // k_shade_emit re-packs q1/q2
            }
        }
    }
    return o;
}

// Warp-aggregated append of the visible Gaussians to the compact list + their records.  Whole warps must call.
__device__ __forceinline__ void append_visible(const Projected& o, const int i, float4* __restrict__ rec,
                                               uint32_t* __restrict__ vis_list, GsDevStatus* __restrict__ status) {
    const int lane = threadIdx.x & 31;
    const unsigned m = __ballot_sync(0xffffffffu, o.vis);
    if (!m) return;
    unsigned long long base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(&status->num_visible, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (o.vis) {
        const uint32_t slot = (uint32_t)base + __popc(m & ((1u << lane) - 1u));
        vis_list[slot] = (uint32_t)i;
        float4* rr = rec + (size_t)GS_REC_V4 * i;
        rr[0] = o.q0;
        rr[1] = o.q1;
    }
}

// One thread per Gaussian, exact path for all of them (the first version of the pass; dense frames run it).
__global__ void __launch_bounds__(kThreads)
k_project_v1(const GsView v, const float* __restrict__ means3D, const float* __restrict__ opacities,
             const float* __restrict__ scales, const float* __restrict__ rotations, const float* __restrict__ cov3D_precomp,
             int* __restrict__ radii, float4* __restrict__ rec, uint32_t* __restrict__ vis_list,
             GsDevStatus* __restrict__ status) {
    __shared__ GsCam cam;
    gs_load_cam(v, &cam);
    const int i = blockIdx.x * kThreads + threadIdx.x;
    Projected o;
    o.vis = false; o.radius = 0;
    if (i < v.P) {
        o = project_exact(i, v, cam, means3D, opacities, scales, rotations, cov3D_precomp);
        radii[i] = o.radius;
    }
    append_visible(o, i, rec, vis_list, status);
}

// Conservative screen test ahead of the exact path: true only when the exact path is CERTAIN to end with an empty tile
// rect (radius 0), from an upper bound on the splat's pixel radius that needs no matrix product:
//   cov2D = A Sigma A^T + 0.3 I with A = J.V3 (2x3);  |a-0.3| <= |A0|^2 s, |c-0.3| <= |A1|^2 s, |b| <= |A0||A1| s with
//   s = ||Sigma||_2;  lambda1 = mid + sqrt(max(0.1, ((a-c)/2)^2 + b^2)) <= max(a,c) + |b| + 0.3163 <= 1.5 ||A||_F^2 s + 0.62;
//   ||A||_F <= ||J||_F ||V3||_2, and ||V3||_2^2 <= vnorm2 = (tr G^8)^(1/8) with G = V3^T V3 (1.147 for a rigid view matrix);
//   s = ||M||_2^2 (Sigma = M^T M, M = S R^T) <= (mod s_max)^2 ||R||_2^2, and for the UN-normalised quaternion the
//   reference feeds in, R(q) = (1 - n) I + n R(q/|q|) with n = |q|^2, so ||R||_2 <= |1 - n| + n (= 1 for a unit q);
//   a precomputed covariance (symmetric or not, definite or not): s <= ||Sigma||_F.
// About 1.3x loose in radius -- most Gaussians behind the near-plane cut are far outside the image anyway (93 % at
// BASELINE config 3).  The 1 % / +2 / +1e-5|px| slacks cover float rounding (incl. the cancellation in mid^2 - det) and
// the reference's double-precision ndc2Pix; NaN or infinite intermediates never reject.
__device__ __forceinline__ bool surely_offscreen(const int i, const float3 p, const float3 t, const GsView& v,
                                                 const GsCam& cam, const float vnorm2, const float3 s, const float4 q,
                                                 const float* __restrict__ cov3D_precomp) {
    const float hx = cam.pm[0] * p.x + cam.pm[4] * p.y + cam.pm[8] * p.z + cam.pm[12];
    const float hy = cam.pm[1] * p.x + cam.pm[5] * p.y + cam.pm[9] * p.z + cam.pm[13];
    const float hw = cam.pm[3] * p.x + cam.pm[7] * p.y + cam.pm[11] * p.z + cam.pm[15];
    const float iw = 1.0f / (hw + 0.0000001f);
    const float px = ((hx * iw + 1.0f) * (float)v.W - 1.0f) * 0.5f;
    const float py = ((hy * iw + 1.0f) * (float)v.H - 1.0f) * 0.5f;
    const float iz = 1.0f / t.z;
    const float limx = 1.3f * v.tan_fovx, limy = 1.3f * v.tan_fovy;
    const float cx = fminf(limx, fmaxf(-limx, t.x * iz)), cy = fminf(limy, fmaxf(-limy, t.y * iz));
    const float J00 = v.focal_x * iz, J11 = v.focal_y * iz;
    const float nJ = J00 * J00 * (1.0f + cx * cx) + J11 * J11 * (1.0f + cy * cy);     // J = [J00 0 -J00 cx; 0 J11 -J11 cy]
    float nS;
    if (cov3D_precomp) {
        float c[6];
#pragma unroll
        for (int k = 0; k < 6; k++) c[k] = cov3D_precomp[6 * i + k];
        nS = sqrtf(c[0] * c[0] + c[3] * c[3] + c[5] * c[5] + 2.f * (c[1] * c[1] + c[2] * c[2] + c[4] * c[4]));
    } else {
        const float n = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
        const float sm = v.scale_modifier * fmaxf(fabsf(s.x), fmaxf(fabsf(s.y), fabsf(s.z))) * (fabsf(1.0f - n) + n);
        nS = sm * sm;
    }
    const float L = 1.52f * (nJ * vnorm2) * nS + 1.0f;
    if (!(L < 1e30f)) return false;                      // overflow or NaN: let the exact path decide
    const float Rb = 3.f * sqrtf(L) + 2.f;
    const float sx = Rb + 1e-5f * fabsf(px), sy = Rb + 1e-5f * fabsf(py);
    // gs_rect: empty when (px + r + 15) / 16 truncates to <= 0 or (px - r) / 16 to >= gx (same in y)
    return (px + sx + 15.f < 0.f) || (px - sx >= 16.f * (float)v.gx) || (py + sy + 15.f < 0.f) || (py - sy >= 16.f * (float)v.gy);
}

// Persistent CTAs, two kinds of rounds: (1) cull round over a block of 256 Gaussians -- every thread tests its own by the
// near plane and the conservative screen test, survivors go into a shared-memory queue; (2) as soon as the queue holds a
// CTA's worth (and once more at the end) the exact path runs over queued Gaussians with every lane busy.  Far from the
// view most blocks queue a handful, so the 600-instruction exact path runs once per ~25 cull rounds instead of once per
// block with one warp; inside the view every block fills the queue and the kernel degenerates to v1 plus the test.
constexpr int kProjQueue = 2 * kThreads;
__global__ void __launch_bounds__(kThreads, 4)
k_project(const GsView v, const float* __restrict__ means3D, const float* __restrict__ opacities,
          const float* __restrict__ scales, const float* __restrict__ rotations, const float* __restrict__ cov3D_precomp,
          int* __restrict__ radii, float4* __restrict__ rec, uint32_t* __restrict__ vis_list,
          GsDevStatus* __restrict__ status) {
    __shared__ GsCam cam;
    __shared__ int s_wcnt[kThreads / 32];
    __shared__ uint32_t s_q[kProjQueue];
    gs_load_cam(v, &cam);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int nblocks = (v.P + kThreads - 1) / kThreads;
    int nq = 0;                                          // queue length, kept identically by every thread
    // upper bound of ||V3||_2^2 of the view matrix for surely_offscreen: (tr G^8)^(1/8), G = V3^T V3
    float vnorm2;
    {
        float G[3][3], G2[3][3], G4[3][3];
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
            for (int c = 0; c < 3; c++)
                G[a][c] = cam.vm[4 * a] * cam.vm[4 * c] + cam.vm[1 + 4 * a] * cam.vm[1 + 4 * c] + cam.vm[2 + 4 * a] * cam.vm[2 + 4 * c];
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
            for (int c = 0; c < 3; c++) G2[a][c] = G[a][0] * G[0][c] + G[a][1] * G[1][c] + G[a][2] * G[2][c];
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
            for (int c = 0; c < 3; c++) G4[a][c] = G2[a][0] * G2[0][c] + G2[a][1] * G2[1][c] + G2[a][2] * G2[2][c];
        float t8 = 0.f;
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
            for (int c = 0; c < 3; c++) t8 += G4[a][c] * G4[a][c];
        // tr G = ||V3||_F^2 bounds it too; it takes over when G^8 leaves the float range (view matrices scaled by < 4e-3
        // or > 1e2 -- nothing a camera produces, but an underflow to 0 must not turn into a radius bound of 0)
        const float trG = G[0][0] + G[1][1] + G[2][2];
        vnorm2 = (t8 > 1e-30f && t8 < 1e30f) ? fminf(trG, sqrtf(sqrtf(sqrtf(t8))) * 1.001f) : trG;
    }

    // exact path over the n queued Gaussians s_q[from .. from + n), n <= kThreads
    auto drain = [&](const int from, const int n) {
        if (wid * 32 < n) {                              // warp-uniform
            Projected o;
            o.vis = false; o.radius = 0;
            int i = 0;
            if (tid < n) {
                i = (int)s_q[from + tid];
                o = project_exact(i, v, cam, means3D, opacities, scales, rotations, cov3D_precomp);
                radii[i] = o.radius;
            }
            append_visible(o, i, rec, vis_list, status);
        }
    };

    // One cull round ahead, every thread has its Gaussian's mean, scale and rotation in flight (unconditionally: the
    // round itself is then a pure ALU chain; the bytes of the half behind the near plane are cheap next to the latency).
    struct Row { float3 p, s; float4 q; };
    auto load_row = [&](const int i) {
        Row r;
        r.p = make_float3(0.f, 0.f, 0.f); r.s = r.p; r.q = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < v.P) {
            r.p = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
            if (!cov3D_precomp) {
                r.s = make_float3(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]);
                r.q = __ldg(reinterpret_cast<const float4*>(rotations) + i);
            }
        }
        return r;
    };
    int b = blockIdx.x;
    Row cur = load_row(b < nblocks ? b * kThreads + tid : v.P);
    for (; b < nblocks; b += gridDim.x) {
        const int i = b * kThreads + tid;
        const Row nxt = load_row(b + (int)gridDim.x < nblocks ? (b + (int)gridDim.x) * kThreads + tid : v.P);
        const float3 p = cur.p;
        bool cand = false;
        if (i < v.P) {
            const float3 t = gs_xf4x3(p, cam.vm);
            // the exact path repeats the near-plane test on its own evaluation of z; this one only has to be no stricter
            const float zerr = 2e-6f * (fabsf(cam.vm[2] * p.x) + fabsf(cam.vm[6] * p.y) + fabsf(cam.vm[10] * p.z) + fabsf(cam.vm[14]));
            if (!(t.z <= GS_NEAR - zerr))                // NaN stays a candidate
                cand = !(t.z > 0.5f * GS_NEAR && surely_offscreen(i, p, t, v, cam, vnorm2, cur.s, cur.q, cov3D_precomp));
            if (!cand) radii[i] = 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, cand);
        if (lane == 0) s_wcnt[wid] = __popc(m);
        __syncthreads();                                 // counts visible; the previous drain has finished reading s_q
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) { const int c = s_wcnt[w]; if (w < wid) before += c; total += c; }
        if (cand) s_q[nq + before + __popc(m & ((1u << lane) - 1u))] = (uint32_t)i;
        nq += total;
        __syncthreads();                                 // queue entries visible; s_wcnt free for the next round
        if (nq >= kThreads) {
            nq -= kThreads;
            drain(nq, kThreads);                         // the newest kThreads entries; the older nq stay queued
        }
        cur = nxt;
    }
    drain(0, nq);
}

// Loads one Gaussian's SH coefficients with every load in flight before the first use, evaluates the colour.
template <int D>
__device__ __forceinline__ void sh_to_rgb(const float* __restrict__ sh, float x, float y, float z, float& cr,
                                          float& cg, float& cb) {
    constexpr int NA = (D + 1) * (D + 1);                // active coefficients
    constexpr int NV = (NA * 3 + 3) / 4;                 // float4 loads (rows are 16-byte aligned when M*3 % 4 == 0)
    float c[NV * 4];
    const float4* s4 = reinterpret_cast<const float4*>(sh);
#pragma unroll
    for (int k = 0; k < NV; k++) {
        const float4 t = __ldg(s4 + k);
        c[4 * k] = t.x; c[4 * k + 1] = t.y; c[4 * k + 2] = t.z; c[4 * k + 3] = t.w;
    }
    float bs[16];
    gs_sh_basis(D, x, y, z, bs);
    cr = bs[0] * c[0]; cg = bs[0] * c[1]; cb = bs[0] * c[2];
#pragma unroll
    for (int k = 1; k < NA; k++) { cr = cr + bs[k] * c[3 * k]; cg = cg + bs[k] * c[3 * k + 1]; cb = cb + bs[k] * c[3 * k + 2]; }
}

// Exclusive scan of the G tile counts by ONE CTA of T threads.  Every thread owns K consecutive tiles (128-bit loads,
// all in flight), scans them in registers, and the block scans the per-thread totals; G <= T * K needs one round (8160
// tiles at 1080p).  Resets the counts to zero so the same array serves as the emission cursors, and mirrors the totals
// to a pinned host slot.  The counts were produced by L2 atomics of other CTAs: read past L1.
template <int T, int K>
__device__ __forceinline__ void cta_tile_scan(const int G, uint32_t* __restrict__ tile_cnt, uint32_t* __restrict__ tile_off,
                                              GsDevStatus* __restrict__ status, GsDevStatus* host_slot, uint32_t* s_warp,
                                              uint32_t* s_carry) {
    static_assert(K % 4 == 0 && T % 32 == 0 && T <= 1024, "scan shape");
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) *s_carry = 0;
    __syncthreads();
    for (int base = 0; base < G; base += T * K) {
        const int t0 = base + tid * K;                   // tile_cnt / tile_off are 256-byte aligned, t0 % 4 == 0
        uint32_t cv[K];
        if (t0 + K <= G) {
#pragma unroll
            for (int k = 0; k < K; k += 4) {
                const uint4 a = __ldcg(reinterpret_cast<const uint4*>(tile_cnt + t0 + k));
                cv[k] = a.x; cv[k + 1] = a.y; cv[k + 2] = a.z; cv[k + 3] = a.w;
            }
        } else {
#pragma unroll
            for (int k = 0; k < K; k++) cv[k] = (t0 + k < G) ? __ldcg(tile_cnt + t0 + k) : 0u;
        }
        uint32_t tot = 0;
#pragma unroll
        for (int k = 0; k < K; k++) { const uint32_t c = cv[k]; cv[k] = tot; tot += c; }   // exclusive, local
        uint32_t x = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = lane < T / 32 ? s_warp[lane] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
            if (lane < T / 32) s_warp[lane] = w;         // inclusive over warps
        }
        __syncthreads();
        const uint32_t carry = *s_carry;
        const uint32_t excl = carry + (x - tot) + (wid ? s_warp[wid - 1] : 0u);
        if (t0 + K <= G) {
#pragma unroll
            for (int k = 0; k < K; k += 4) {
                *reinterpret_cast<uint4*>(tile_off + t0 + k) = make_uint4(excl + cv[k], excl + cv[k + 1], excl + cv[k + 2], excl + cv[k + 3]);
                *reinterpret_cast<uint4*>(tile_cnt + t0 + k) = make_uint4(0u, 0u, 0u, 0u);
            }
        } else {
#pragma unroll
            for (int k = 0; k < K; k++)
                if (t0 + k < G) { tile_off[t0 + k] = excl + cv[k]; tile_cnt[t0 + k] = 0u; }
        }
        __syncthreads();
        if (tid == T - 1) *s_carry = excl + tot;
        __syncthreads();
    }
    if (tid == 0) {
        const uint32_t total = *s_carry;
        tile_off[G] = total;
        status->num_pairs = total;
        if (host_slot) {
            host_slot->num_rendered = *reinterpret_cast<volatile unsigned long long*>(&status->num_rendered);
            host_slot->num_pairs = total;
            host_slot->num_visible = *reinterpret_cast<volatile unsigned long long*>(&status->num_visible);
            __threadfence_system();
            host_slot->overflow = 0xC0FFEEu;            // "written" marker, checked by gs_forward_counts
        }
    }
}

// the scan as a kernel of its own, for empty models (no k_count_tiles launch)
constexpr int kScanT = 1024, kScanK = 8;
__global__ void __launch_bounds__(kScanT)
k_tile_scan(int G, uint32_t* __restrict__ tile_cnt, uint32_t* __restrict__ tile_off, GsDevStatus* __restrict__ status,
            GsDevStatus* host_slot) {
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    cta_tile_scan<kScanT, kScanK>(G, tile_cnt, tile_off, status, host_slot, s_warp, &s_carry);
}

__global__ void __launch_bounds__(kThreads, 6)
k_count_tiles(const GsView v, const int* __restrict__ radii, const float4* __restrict__ rec,
              const uint32_t* __restrict__ vis_list, uint32_t* __restrict__ hitmask, uint32_t* __restrict__ tile_cnt,
              GsDevStatus* __restrict__ status, uint32_t* __restrict__ tile_off, GsDevStatus* host_slot, const bool scan_here) {
    __shared__ CandShared S;
    const uint32_t nvis = (uint32_t)status->num_visible;
    const int CH = vis_chunk(nvis);
    unsigned long long rendered = 0;                      // thread 0: sum of the rect areas this CTA has seen
    for (uint32_t chunk = blockIdx.x * CH; chunk < nvis; chunk += gridDim.x * CH) {
        const uint32_t c = chunk + threadIdx.x;
        uint32_t area = 0;
        if (threadIdx.x < CH && c < nvis) {
            const uint32_t i = vis_list[c];
            const float4* rr = rec + (size_t)GS_REC_V4 * i;
            const float4 q0 = __ldg(rr), q1 = __ldg(rr + 1);   // k_project: (x,y,A,B), (C, opacity, depth, thr)
            const int4 rect = gs_rect(q0.x, q0.y, radii[i], v.gx, v.gy);
            area = (uint32_t)((rect.z - rect.x) * (rect.w - rect.y));
            const int t = threadIdx.x;
            S.mx[t] = q0.x; S.my[t] = q0.y; S.A[t] = q0.z; S.B[t] = q0.w; S.C[t] = q1.x; S.thr[t] = q1.w;
            S.rx[t] = rect.x; S.ry[t] = rect.y; S.rw[t] = rect.z - rect.x; S.p0[t] = area; S.bits[t] = 0u;
        }
        const uint32_t total = cta_scan_areas(S, area, CH);
        cta_for_each_candidate(S, total, CH, [&](bool valid, int cc, int r, int tx, int ty) {
            const bool hit = valid && gs_tile_hit(S.mx[cc], S.my[cc], S.A[cc], S.B[cc], S.C[cc], S.thr[cc], tx, ty);
            const uint32_t tile = (uint32_t)(ty * v.gx + tx);
            int n; bool leader; unsigned peers;
            tile_peers(hit, tile, n, leader, peers);
            if (leader) atomicAdd(&tile_cnt[tile], (uint32_t)n);
            if (hit && S.p0[cc] <= kBitRect) atomicOr(&S.bits[cc], 1u << r);
        });
        __syncthreads();
        if (threadIdx.x < CH && c < nvis && area <= kBitRect) hitmask[c] = S.bits[threadIdx.x];
        if (threadIdx.x == 0) rendered += total;         // num_rendered keeps the reference's meaning (rasterizer_impl.cu:278-282)
        __syncthreads();
    }
    if (threadIdx.x == 0 && rendered) atomicAdd(&status->num_rendered, rendered);
    if (!scan_here) return;
    // The last CTA to finish scans the histogram (k_tile_scan's work without its launch): every CTA publishes its
    // atomics, then takes a ticket.
    __shared__ bool s_last;
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    __threadfence();
    __syncthreads();                                     // this CTA's tile_cnt atomics are all issued and ordered
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(&status->pad, 1u) == gridDim.x - 1;
        __threadfence();
    }
    __syncthreads();
    if (!s_last) return;
    cta_tile_scan<kThreads, kFoldK>(v.gx * v.gy, tile_cnt, tile_off, status, host_slot, s_warp, &s_carry);
}

// After the scan (off the host's critical path): SH -> RGB for the visible Gaussians, final record + zeroed
// accumulator, and emission of the (tile, Gaussian) pairs into the tile buckets.
// SH rows (192 B at M = 16, the bulk of this kernel's input) arrive by TMA when they can: every thread issues one
// cp.async.bulk for its own Gaussian's row into a padded shared-memory slot (52 floats apart: conflict-free 128-bit
// reads), one mbarrier per CTA counts the bytes, and the rest of the per-Gaussian loads (record, mean, radius) are in
// flight meanwhile.  Rows of other widths / alignments take the direct 128-bit or scalar loads.
constexpr int kShRow = 52;            // shared-memory row stride in floats

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// colour from a Gaussian's SH row staged in shared memory (generic 128-bit loads; only the active coefficients)
template <int D>
__device__ __forceinline__ void sh_smem_to_rgb(const float* row, float x, float y, float z, float& cr, float& cg, float& cb) {
    constexpr int NA = (D + 1) * (D + 1);
    constexpr int NV = (NA * 3 + 3) / 4;
    float c[NV * 4];
    const float4* s4 = reinterpret_cast<const float4*>(row);
#pragma unroll
    for (int k = 0; k < NV; k++) {
        const float4 t = s4[k];
        c[4 * k] = t.x; c[4 * k + 1] = t.y; c[4 * k + 2] = t.z; c[4 * k + 3] = t.w;
    }
    float bs[16];
    gs_sh_basis(D, x, y, z, bs);
    cr = bs[0] * c[0]; cg = bs[0] * c[1]; cb = bs[0] * c[2];
#pragma unroll
    for (int k = 1; k < NA; k++) { cr = cr + bs[k] * c[3 * k]; cg = cg + bs[k] * c[3 * k + 1]; cb = cb + bs[k] * c[3 * k + 2]; }
}

__global__ void __launch_bounds__(kThreads)
k_shade_emit(const GsView v, const float* __restrict__ means3D, const float* __restrict__ shs,
             const float* __restrict__ colors_precomp, const int* __restrict__ radii, float4* __restrict__ rec,
             float4* __restrict__ acc, const uint32_t* __restrict__ vis_list, const uint32_t* __restrict__ hitmask,
             const uint32_t* __restrict__ tile_off, uint32_t* __restrict__ tile_cur, GsDevStatus* __restrict__ status,
             unsigned long long* __restrict__ keys, long long capacity, const bool shaded, const bool use_tma) {
    extern __shared__ __align__(16) float s_sh[];                    // kChunkMax x kShRow floats when use_tma
    const bool overflow = (long long)status->num_pairs > capacity;   // device-side guard: nothing is binned then,
    if (blockIdx.x == 0 && threadIdx.x == 0) {                       // the host re-renders with a larger buffer
        if (overflow) status->overflow = 1u;
        else { status->n_big = 0u; status->n_mid = 0u; }
    }
    __shared__ CandShared S;
    __shared__ __align__(16) float s_campos[4];         // own 16-byte slot: the compiler reads it with one 128-bit load
    __shared__ __align__(8) unsigned long long s_bar;
    const uint32_t bar = smem_addr(&s_bar);
    if (threadIdx.x < 4) s_campos[threadIdx.x] = threadIdx.x < 3 ? __ldg(v.campos + threadIdx.x) : 0.f;
    const uint32_t nvis = (uint32_t)status->num_visible;
    const int CH = vis_chunk(nvis);
    // TMA staging pays when the rows are (nearly) consecutive and every thread has one: the many-visible regime
    const bool tma = use_tma && !shaded && CH == kChunkMax;
    if (tma && threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const bool aligned = ((v.M * 3) & 3) == 0;
    uint32_t parity = 0;
    for (uint32_t chunk = blockIdx.x * CH; chunk < nvis; chunk += gridDim.x * CH) {
        const uint32_t c = chunk + threadIdx.x;
        const bool active = threadIdx.x < CH && c < nvis;
        uint32_t i = 0;
        float* my_sh = s_sh + threadIdx.x * kShRow;
        if (tma) {
            if (threadIdx.x == 0) {
                const uint32_t nact = min((uint32_t)CH, nvis - chunk);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(nact * 192u) : "memory");
            }
            if (active) {
                i = vis_list[c];
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_addr(my_sh)), "l"(shs + (size_t)i * 48), "r"(192), "r"(bar) : "memory");
            }
        } else if (active) {
            i = vis_list[c];
        }
        uint32_t area = 0;
        if (active) {
            float4* rr = rec + (size_t)GS_REC_V4 * i;
            const float4 q0 = rr[0];
            float4 q1 = rr[1];
            float depth, thr;
            const float4 q2old = rr[2];
            const int radius = radii[i];
            // first render of this frame: q1 = (C, opacity, depth, thr) from k_project.  A re-render after a capacity
            // overflow (`shaded`, set by the host) finds the final record layout already in place.
            if (!shaded) {
                depth = q1.z; thr = q1.w;
                float r_, g_, b_;
                uint32_t clamped = 0;
                if (colors_precomp) {
                    r_ = colors_precomp[3 * i]; g_ = colors_precomp[3 * i + 1]; b_ = colors_precomp[3 * i + 2];
                } else {                                 // forward.cu:20-71
                    const float3 p = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
                    float3 d = make_float3(p.x - s_campos[0], p.y - s_campos[1], p.z - s_campos[2]);
                    const float len = sqrtf(d.x * d.x + d.y * d.y + d.z * d.z);
                    d.x = d.x / len; d.y = d.y / len; d.z = d.z / len;
                    const float* sh = shs + (size_t)i * v.M * 3;
                    float cr, cg, cb;
                    if (tma) {
                        uint32_t done = 0;               // the CTA's SH rows have landed when this phase completes
                        while (!done) {
                            asm volatile("{.reg .pred p;\n\t"
                                         "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                                         "selp.u32 %0, 1, 0, p;}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
                        }
                        switch (v.D) {
                            case 0: sh_smem_to_rgb<0>(my_sh, d.x, d.y, d.z, cr, cg, cb); break;
                            case 1: sh_smem_to_rgb<1>(my_sh, d.x, d.y, d.z, cr, cg, cb); break;
                            case 2: sh_smem_to_rgb<2>(my_sh, d.x, d.y, d.z, cr, cg, cb); break;
                            default: sh_smem_to_rgb<3>(my_sh, d.x, d.y, d.z, cr, cg, cb); break;
                        }
                    } else if (aligned) {
                        switch (v.D) {
                            case 0: sh_to_rgb<0>(sh, d.x, d.y, d.z, cr, cg, cb); break;
                            case 1: sh_to_rgb<1>(sh, d.x, d.y, d.z, cr, cg, cb); break;
                            case 2: sh_to_rgb<2>(sh, d.x, d.y, d.z, cr, cg, cb); break;
                            default: sh_to_rgb<3>(sh, d.x, d.y, d.z, cr, cg, cb); break;
                        }
                    } else {
                        float bs[16];
                        gs_sh_basis(v.D, d.x, d.y, d.z, bs);
                        cr = bs[0] * sh[0]; cg = bs[0] * sh[1]; cb = bs[0] * sh[2];
                        const int na = (v.D + 1) * (v.D + 1);
                        for (int k = 1; k < na; k++) { cr = cr + bs[k] * sh[3 * k]; cg = cg + bs[k] * sh[3 * k + 1]; cb = cb + bs[k] * sh[3 * k + 2]; }
                    }
                    cr += 0.5f; cg += 0.5f; cb += 0.5f;
                    clamped = (cr < 0.f ? 1u : 0u) | (cg < 0.f ? 2u : 0u) | (cb < 0.f ? 4u : 0u);
                    r_ = fmaxf(cr, 0.f); g_ = fmaxf(cg, 0.f); b_ = fmaxf(cb, 0.f);
                }
                q1 = make_float4(q1.x, q1.y, r_, g_);
                rr[1] = q1;
                rr[2] = make_float4(b_, depth, __uint_as_float(clamped), thr);
                float4* aa = acc + (size_t)3 * i;
                const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
                aa[0] = z4; aa[1] = z4;
                aa[2] = make_float4(0.f, __uint_as_float(clamped), 0.f, __uint_as_float(c));   // a2.y = SH clamp bits
                                                                                                 // a2.w = compact slot
            } else {
                depth = q2old.y; thr = q2old.w;
            }
            const int4 rect = gs_rect(q0.x, q0.y, radius, v.gx, v.gy);   // same recomputation as rasterizer_impl.cu:91
            const int rw = rect.z - rect.x;
            area = overflow ? 0u : (uint32_t)(rw * (rect.w - rect.y));
            const int t = threadIdx.x;
            S.mx[t] = q0.x; S.my[t] = q0.y; S.A[t] = q0.z; S.B[t] = q0.w; S.C[t] = q1.x; S.thr[t] = thr;
            S.rx[t] = rect.x; S.ry[t] = rect.y; S.rw[t] = rw;
            S.p0[t] = __float_as_uint(depth); S.p1[t] = i;
            // rects of up to kBitRect tiles: the histogram pass left its decisions (same tiles, same order); larger ones
            // repeat the test (same machine code on the same operands: gs_tile_hit)
            S.bits[t] = (area != 0u && area <= kBitRect) ? hitmask[c] : 0u;
        }
        const uint32_t total = cta_scan_areas(S, area, CH);
        cta_for_each_candidate(S, total, CH, [&](bool valid, int cc, int r, int tx, int ty) {
            bool hit = false;
            if (valid) {
                const bool big = (S.cum[cc + 1] - S.cum[cc]) > (uint32_t)kBitRect;
                hit = big ? gs_tile_hit(S.mx[cc], S.my[cc], S.A[cc], S.B[cc], S.C[cc], S.thr[cc], tx, ty)
                          : ((S.bits[cc] >> r) & 1u) != 0u;
            }
            const uint32_t tile = (uint32_t)(ty * v.gx + tx);
            int n; bool leader; unsigned peers;
            const int rank = tile_peers(hit, tile, n, leader, peers);
            uint32_t basepos = 0;
            if (leader) basepos = tile_off[tile] + atomicAdd(&tile_cur[tile], (uint32_t)n);   // one atomic per (warp, tile)
            basepos = __shfl_sync(0xffffffffu, basepos, __ffs(peers) - 1);
            if (hit) keys[basepos + rank] = ((unsigned long long)S.p0[cc] << 32) | S.p1[cc];
        });
        parity ^= 1u;
        __syncthreads();
    }
}

__global__ void k_mark_visible(int P, const float* __restrict__ means3D, const float* __restrict__ vm,
                               uint8_t* __restrict__ present) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float3 p = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
    const float z = vm[2] * p.x + vm[6] * p.y + vm[10] * p.z + vm[14];
    present[i] = z > GS_NEAR ? 1 : 0;
}

}  // namespace

void gs_launch_project(const GsView& v, const float* means3D, const float* opacities, const float* scales,
                       const float* rotations, const float* cov3D_precomp, int* radii, float4* rec,
                       uint32_t* vis_list, GsDevStatus* status, bool dense_hint, cudaStream_t s) {
    const int grid = (v.P + kThreads - 1) / kThreads;
    // most of the model was inside the previous view of this context: the screen pre-test would reject next to nothing
    // -- skip it (same results either way)
    const int pgrid = grid < g_gs_num_sms * 4 ? grid : g_gs_num_sms * 4;      // persistent: 4 CTAs of <= 64 registers per SM
    if (dense_hint) k_project_v1<<<grid, kThreads, 0, s>>>(v, means3D, opacities, scales, rotations, cov3D_precomp, radii, rec, vis_list, status);
    else k_project<<<pgrid, kThreads, 0, s>>>(v, means3D, opacities, scales, rotations, cov3D_precomp, radii, rec, vis_list, status);
}
void gs_launch_count_tiles(const GsView& v, int num_sms, const int* radii, const float4* rec, const uint32_t* vis_list,
                           uint32_t* hitmask, uint32_t* tile_cnt, GsDevStatus* status, uint32_t* tile_off,
                           GsDevStatus* host_slot, cudaStream_t s) {
    const int need = (v.P + kChunkMin - 1) / kChunkMin;
    const int grid = need < num_sms * 8 ? need : num_sms * 8;
    k_count_tiles<<<grid, kThreads, 0, s>>>(v, radii, rec, vis_list, hitmask, tile_cnt, status, tile_off, host_slot,
                                            true);
}
void gs_launch_tile_scan(int G, uint32_t* tile_cnt, uint32_t* tile_off, GsDevStatus* status, GsDevStatus* host_slot,
                         cudaStream_t s) {
    k_tile_scan<<<1, kScanT, 0, s>>>(G, tile_cnt, tile_off, status, host_slot);
}
void gs_preprocess_init() {
    cudaFuncSetAttribute(k_shade_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, kChunkMax * kShRow * (int)sizeof(float));
}
void gs_launch_shade_emit(const GsView& v, int num_sms, const float* means3D, const float* shs,
                          const float* colors_precomp, const int* radii, float4* rec, float4* acc,
                          const uint32_t* vis_list, const uint32_t* hitmask, const uint32_t* tile_off, uint32_t* tile_cur,
                          GsDevStatus* status, unsigned long long* keys, long long capacity, bool shaded, bool dense_hint,
                          cudaStream_t s) {
    const int need = (v.P + kChunkMin - 1) / kChunkMin;
    // TMA staging of the SH rows: 16 stored coefficients (192-byte rows, 16-byte aligned like the base pointer).  The
    // kernel uses it only when most Gaussians are visible; `dense_hint` (the previous frame on this context) decides
    // whether the launch reserves the 53 KB staging buffer at all -- either way the result is the same.
    const bool use_tma = dense_hint && shs && !colors_precomp && v.M == 16;
    const size_t smem = use_tma ? (size_t)kChunkMax * kShRow * sizeof(float) : 0;
    const int per_sm = use_tma ? 4 : 8;                  // 53 KB of shared memory per CTA with the staging buffer
    const int grid = need < num_sms * per_sm ? need : num_sms * per_sm;
    k_shade_emit<<<grid, kThreads, smem, s>>>(v, means3D, shs, colors_precomp, radii, rec, acc, vis_list, hitmask, tile_off,
                                              tile_cur, status, keys, capacity, shaded, use_tma);
}
void gs_launch_mark_visible(int P, const float* means3D, const float* vm, uint8_t* present, cudaStream_t s) {
    k_mark_visible<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, vm, present);
}
