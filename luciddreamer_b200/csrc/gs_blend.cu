// Tile compositing, forward (sm_90a); the backward tile pass is gs_blend_bwd.cu.
//
// k_blend_fwd replaces RAST/cuda_rasterizer/forward.cu:261-391 (renderCUDA): front-to-back alpha compositing of
//   colour + depth per 16x16 tile, same formulas per (pixel, splat).
// k_blend_bwd (gs_blend_bwd.cu) replaces backward.cu:399-586 (renderCUDA backward), same formulas per (pixel, splat).
//
// Both kernels are instruction-issue bound (a few bytes of DRAM traffic per (pixel, splat)), so the
// design minimises issued instructions per (pixel, splat) evaluation:
//  * one CTA of 64 threads per tile; a warp owns a 16x8 pixel block and every thread FOUR pixels of one column
//    (x, y), (x, y+2), (x, y+4), (x, y+6), held as two float2 PAIRS: all per-pixel arithmetic is written
//    on pairs (fma2 / mul2 / add2, one FFMA / FMUL / FADD per pixel on sm_90; per-splat scalars ride along as
//    broadcast operands);
//  * the per-splat record (xy, conic, opacity, rgb, depth) is fetched ONCE per (tile, splat) with 128-bit loads
//    into shared memory; the staging thread also tests its splat against the tile's two 16x8 blocks (exact
//    ellipse-vs-box test) and the warps ballot the results into a bit mask per block, walked with one FLO per hit;
//  * per-splat FAST-PATH eligibility is decided once at staging (warp-uniform): opacity <= 0.99 (the
//    min(0.99, alpha) clamp of forward.cu:343 can never bind) and a well-conditioned positive-definite conic
//    (power <= 0 holds with a 10x margin over fp32 rounding, so forward.cu:336's `power > 0` test can never
//    fire).  Eligible splats skip both per-pixel tests; everything else takes the generic path, which is the
//    reference's test sequence verbatim;
//  * exp(): ex2.approx of the log2-scaled power (conic pre-multiplied at staging).  alpha is compared against
//    1/255; inside a band of 1e-7 around that threshold a thread re-evaluates its four alphas with expf and
//    the reference's expression (generic path), so the skip decision is the reference's.  Forward and
//    backward run the SAME instruction sequence up to that decision, hence skip exactly the same
//    (pixel, splat) pairs;
//  * backward: the reference issues 9 global float atomicAdds per contributing (pixel, splat); here the 9 partials
//    of the four pixels are summed in registers, reduced across the warp through shared memory, and leave the CTA as
//    128-bit vector reductions: one per (tile, splat).  1/(1-alpha) is a single MUFU.RCP (the gradient tolerance is
//    1e-3 relative).  gs_blend_bwd.cu holds the pass and its reduction order.
// k_tile_partials (deterministic backward, opt-in; gs_blend_bwd.cu) is k_blend_bwd with the reductions replaced by plain
//   stores of the same nine values per list position; gs_det_bwd.cu sums them per Gaussian in a fixed order.

#include "gs_blend.cuh"

namespace {

constexpr int kBatch = 128;           // splats staged per round
constexpr int kWords = kBatch / 32;

// the thread's pixels as packed pairs: pair h holds image rows pyb + 4h and pyb + 4h + 2
template <int NH> struct FwdPix {
    float2 T[NH];                     // transmittance in front of the next splat; frozen once the pixel is dead
    float2 nam[NH];                   // -1/255 while the pixel is live; -inf once it terminated (T < 1e-4) or if it
                                      // lies outside the image: a + nam < 0 then fails the alpha test for every splat
    float2 C0[NH], C1[NH], C2[NH], D[NH], acc[NH];
    uint32_t last[2 * NH];
};

// forward.cu:330-369, generic path: the reference's full test sequence per pixel (power > 0, min(0.99, alpha),
// alpha < 1/255, T < 1e-4).  Taken by splats that are not fast-path eligible, by threads with an alpha in the band and
// whenever a pixel of the warp is about to terminate.
template <int NH>
__device__ __forceinline__ void fwd_generic(FwdPix<NH>& P, const SRec& r, const float dx, const float2* dy, const float2* p,
                                            const float2* a, const bool band, const uint32_t pos1,
                                            const float4* __restrict__ rec) {
    // in the band around 1/255, and for every splat that is not fast-path eligible (ill-conditioned conics: the
    // factored exponent rounds differently from the reference's expression, and the difference is amplified by the
    // cancellation inside `power`), the decision operands are re-evaluated in the reference's own operation order
    float alpha[2 * NH], power[2 * NH];
#pragma unroll
    for (int q = 0; q < 2 * NH; q++) { alpha[q] = GS_Q(a, q); power[q] = GS_Q(p, q); }
    if (band || r.generic) exact_eval<NH>(r, dx, dy, rec, power, alpha);
#pragma unroll
    for (int q = 0; q < 2 * NH; q++) {
        float& T = GS_Q(P.T, q);
        const bool live = GS_Q(P.nam, q) > -1.f;
        const float al = fminf(0.99f, alpha[q]);
        const bool ok = live && !(power[q] > 0.0f) && !(al < kAlphaMin);
        const float test_T = T * (1.f - al);
        const bool low = test_T < 0.0001f;                // forward.cu:348-352
        if (ok && !low) {
            const float w = al * T;                       // one weight for colour, depth and coverage
            GS_Q(P.C0, q) += r.b.z * w;
            GS_Q(P.C1, q) += r.b.w * w;
            GS_Q(P.C2, q) += r.c.x * w;
            GS_Q(P.D, q) += r.c.y * w;
            GS_Q(P.acc, q) += w;
            P.last[q] = pos1;
            T = test_T;
        }
        if (ok && low) GS_Q(P.nam, q) = kNegInf;          // done = true: T stays, nothing behind contributes
    }
}

template <int NH, int OCC>
__global__ void __launch_bounds__(Geo<NH>::NT, OCC)
k_blend_fwd(const GsView v, const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ list,
            const float4* __restrict__ rec, const GsDevStatus* __restrict__ status, long long capacity,
            float* __restrict__ final_T, uint32_t* __restrict__ n_contrib, float* __restrict__ out_color,
            float* __restrict__ out_depth) {
    constexpr int NW = Geo<NH>::NW, NQ = Geo<NH>::NQ;
    if ((long long)status->num_pairs > capacity) return;
    __shared__ SRec sRec[kBatch];
    __shared__ uint32_t sMask[NW][kWords];               // [pixel strip][32-splat word], bit-reversed
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const float bg0 = __ldg(v.bg), bg1 = __ldg(v.bg + 1), bg2 = __ldg(v.bg + 2);
    const int tile = blockIdx.y * v.gx + blockIdx.x;
    const int tx0 = blockIdx.x * GS_TILE, ty0 = blockIdx.y * GS_TILE;
    const uint32_t px = tx0 + (lane & 15);
    const uint32_t pyb = ty0 + Geo<NH>::RW * wid + (lane >> 4);    // rows pyb + 2q
    const float pixx = (float)px;
    float2 npy[NH];
#pragma unroll
    for (int h = 0; h < NH; h++) npy[h] = make_float2(-(float)(pyb + 4 * h), -(float)(pyb + 4 * h + 2));
    const uint32_t beg = tile_off[tile], end = tile_off[tile + 1];
    const int n = (int)(end - beg);

    FwdPix<NH> P;
#pragma unroll
    for (int q = 0; q < NQ; q++) {
        const bool in = px < (uint32_t)v.W && (pyb + 2 * q) < (uint32_t)v.H;
        GS_Q(P.T, q) = 1.0f;
        GS_Q(P.nam, q) = in ? -kAlphaMin : kNegInf;
        GS_Q(P.C0, q) = 0.f; GS_Q(P.C1, q) = 0.f; GS_Q(P.C2, q) = 0.f; GS_Q(P.D, q) = 0.f;
        GS_Q(P.acc, q) = 0.000001f; P.last[q] = 0u;
    }
    auto all_dead = [&]() {
        float m = fmaxf(P.nam[0].x, P.nam[0].y);
        if (NH == 2) m = fmaxf(m, fmaxf(P.nam[NH - 1].x, P.nam[NH - 1].y));
        return m < -1.f;
    };

    for (int base = 0; base < n; base += kBatch) {
        if (__syncthreads_and(all_dead())) break;
        const int cnt = min(kBatch, n - base);
        stage_batch<NH, kBatch>(sRec, sMask, list, rec, beg, cnt, tx0, ty0, [&](int j) { return base + j; });
        __syncthreads();
#pragma unroll 1
        for (int k = 0; k < kWords; k++) {
            uint32_t bits = sMask[wid][k];
            if (bits == 0) continue;
            if (__all_sync(0xffffffffu, all_dead())) break;
            while (bits) {
                const int lz = __clz(bits);
                bits &= ~(0x80000000u >> lz);
                const int j = 32 * k + lz;
                const SRec& r = sRec[j];
                const uint32_t pos1 = (uint32_t)(base + j + 1);
                const float dx = r.a.x - pixx;
                float2 dy[NH], p[NH], g[NH], a[NH], d[NH];
#pragma unroll
                for (int h = 0; h < NH; h++) dy[h] = add2(bc(r.a.y), npy[h]);
                const bool band = eval_alpha<NH>(r, dx, dy, P.nam, p, g, a, d);
                // fast path: alpha = a (no clamp can bind), contributes <=> a >= 1/255 on a live pixel <=> d >= 0
                // (forward.cu:336-346).  A pixel that does not contribute runs with alpha = 0: test_T = T exactly.
                float2 ae[NH], tT[NH];
                bool okq[NQ];
#pragma unroll
                for (int q = 0; q < NQ; q++) {
                    okq[q] = GS_Q(d, q) >= 0.f;
                    GS_Q(ae, q) = okq[q] ? GS_Q(a, q) : 0.f;
                }
#pragma unroll
                for (int h = 0; h < NH; h++) {
                    const float2 om = fma2(ae[h], bc(-1.f), bc(1.f));     // 1 - alpha
                    tT[h] = mul2(P.T[h], om);                             // test_T = T * (1 - alpha)
                }
                float tmin = fminf(tT[0].x, tT[0].y);
                if (NH == 2) tmin = fminf(tmin, fminf(tT[NH - 1].x, tT[NH - 1].y));
                // a pixel about to terminate (forward.cu:348-352; dead pixels keep T >= 1e-4 and never trigger), an
                // alpha in the band or an ineligible splat: this thread takes the reference's sequence for its pixels
                if (band || tmin < 0.0001f || r.generic) {
                    fwd_generic<NH>(P, r, dx, dy, p, a, band, pos1, rec);
                    continue;
                }
#pragma unroll
                for (int q = 0; q < NQ; q++) P.last[q] = okq[q] ? pos1 : P.last[q];
#pragma unroll
                for (int h = 0; h < NH; h++) {
                    const float2 w = mul2(ae[h], P.T[h]);                 // alpha * T
                    P.T[h] = tT[h];
                    P.C0[h] = fma2(bc(r.b.z), w, P.C0[h]);
                    P.C1[h] = fma2(bc(r.b.w), w, P.C1[h]);
                    P.C2[h] = fma2(bc(r.c.x), w, P.C2[h]);
                    P.D[h] = fma2(bc(r.c.y), w, P.D[h]);
                    P.acc[h] = add2(P.acc[h], w);
                }
            }
        }
    }
    const size_t HW = (size_t)v.H * v.W;
#pragma unroll
    for (int q = 0; q < NQ; q++) {
        const uint32_t py = pyb + 2 * q;
        if (px < (uint32_t)v.W && py < (uint32_t)v.H) {
            const uint32_t pix_id = (uint32_t)v.W * py + px;
            const float T = GS_Q(P.T, q);
            final_T[pix_id] = T;
            n_contrib[pix_id] = P.last[q];
            out_color[pix_id] = GS_Q(P.C0, q) + T * bg0;
            out_color[HW + pix_id] = GS_Q(P.C1, q) + T * bg1;
            out_color[2 * HW + pix_id] = GS_Q(P.C2, q) + T * bg2;
            out_depth[pix_id] = (GS_Q(P.acc, q) > 0.5f) ? GS_Q(P.D, q) / GS_Q(P.acc, q) : 0.f;
        }
    }
}

}  // namespace

int g_gs_num_sms = 132;           // H100 SXM; replaced by the device's count when a context is created

// 16x4 strips (4 warps per tile) when 16x8 blocks would leave the SMs with fewer than ~20 resident warps
bool gs_blend_use_strips(const GsView& v) {
    return (long long)v.gx * v.gy * 2 < (long long)g_gs_num_sms * 20;
}

void gs_launch_blend_fwd(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                         const GsDevStatus* status, long long capacity, float* final_T, uint32_t* n_contrib,
                         float* out_color, float* out_depth, cudaStream_t s) {
    dim3 grid(v.gx, v.gy);
    // CTAs per SM the register allocation aims at: 14 (72 registers, 28 warps per SM); 12 (80 registers) measured the same
    // on config 3 (H100 SXM, 400 W limit: 0.127 vs 0.128 ms)
    if (gs_blend_use_strips(v))
        k_blend_fwd<1, 6><<<grid, Geo<1>::NT, 0, s>>>(v, tile_off, list, rec, status, capacity, final_T, n_contrib, out_color, out_depth);
    else
        k_blend_fwd<2, 14><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, status, capacity, final_T, n_contrib, out_color, out_depth);
}
