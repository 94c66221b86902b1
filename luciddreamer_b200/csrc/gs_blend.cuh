// Device pieces shared by the tile-compositing passes, forward (gs_blend.cu) and backward (gs_blend_bwd.cu): the warp
// geometries, the staged splat record, FP32 pair arithmetic, staging with the per-strip hit masks, and the alpha
// evaluation both passes run up to the same skip decision.  See gs_blend.cu for the design.
#pragma once

#include "gs_common.cuh"

namespace {

// Two geometries, chosen per launch by the number of tiles (gs_blend_use_strips):
//   NH = 2  a warp owns a 16x8 block, a thread FOUR pixels (two float2 pairs); 2 warps (64 threads) per tile
//   NH = 1  a warp owns a 16x4 strip, a thread TWO pixels (one pair); 4 warps (128 threads) per tile -- twice the warps
//           for images with few tiles (512x512: 1024 tiles would leave the SMs at 14 resident warps), finer culling
template <int NH> struct Geo {
    static constexpr int RW = 4 * NH;             // pixel rows per warp
    static constexpr int NW = 16 / RW;            // warps per tile
    static constexpr int NT = 32 * NW;            // threads per CTA
    static constexpr int NQ = 2 * NH;             // pixels per thread
};

struct __align__(16) SRec {           // shared-memory copy of a splat record
    float4 a;                         // x, y, A2 = -0.5 log2e conic_a, B2 = -log2e conic_b
    float4 b;                         // C2 = -0.5 log2e conic_c, opacity, r, g
    float2 c;                         // b, depth
    uint32_t id;
    uint32_t generic;                 // != 0: not eligible for the fast path
};

constexpr float kHalfLog2e = -0.5f * 1.4426950408889634f;     // staged conic scale (see stage_batch)
constexpr float kAlphaMin = 1.0f / 255.0f;
constexpr float kBand = 1e-7f;
constexpr float kNegInf = -__builtin_huge_valf();

// ---- FP32 pairs: two pixels per call, one FFMA / FMUL / FADD per pixel (sm_90 has no packed FP32 instructions).
// The _rn intrinsics round every product and sum on its own: the compiler may not contract a mul2 + add2 into an fma.
__device__ __forceinline__ float2 fma2(const float2 a, const float2 b, const float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(const float2 a, const float2 b) {
    return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 add2(const float2 a, const float2 b) {
    return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 bc(const float s) { return make_float2(s, s); }
__device__ __forceinline__ float ex2_approx(const float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(const float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// NW-bit mask: which of the tile's 16 x RW pixel strips the splat can touch
template <int NH>
__device__ __forceinline__ uint32_t strip_mask(const float4 a, const float4 b, const float thr, int tx0, int ty0) {
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < Geo<NH>::NW; w++) {
        const float x0 = (float)tx0, y0 = (float)(ty0 + Geo<NH>::RW * w);
        if (gs_box_hit(a.x, a.y, a.z, a.w, b.x, thr, x0, y0, x0 + 15.f, y0 + (float)(Geo<NH>::RW - 1))) m |= 1u << w;
    }
    return m;
}

// Stages up to KB splats into shared memory and publishes the per-strip hit masks.
// slot j of the batch holds list position pos(j).  Mask words are bit-REVERSED (slot 32k+i -> bit 31-i) so the
// traversal finds the next slot with one FLO (count-leading-zeros).  All threads must call.  A batch smaller than the
// CTA (KB < NT) is staged by its first KB / 32 warps.
template <int NH, int KB, typename PosFn>
__device__ __forceinline__ void stage_batch(SRec* sRec, uint32_t (*sMask)[KB / 32], const uint32_t* __restrict__ list,
                                            const float4* __restrict__ rec, uint32_t beg, int cnt, int tx0, int ty0,
                                            PosFn pos_of) {
    constexpr int NW = Geo<NH>::NW, NT = Geo<NH>::NT;
    constexpr int NR = KB >= NT ? KB / NT : 1;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int h = 0; h < NR; h++) {
        const int j = tid + h * NT;
        uint32_t m = 0;
        if (j < cnt) {
            const uint32_t id = list[beg + pos_of(j)];
            const float4* r = rec + (size_t)GS_REC_V4 * id;
            const float4 a = __ldg(r), b = __ldg(r + 1), c = __ldg(r + 2);
            // the conic is staged pre-multiplied for the exponent in base 2:
            //   log2(e) * power = A2 dx dx + C2 dy dy + B2 dx dy,  A2 = -0.5 log2e A, C2 = -0.5 log2e C, B2 = -log2e B
            SRec s; s.a = make_float4(a.x, a.y, a.z * kHalfLog2e, a.w * (2.f * kHalfLog2e));
            s.b = make_float4(b.x * kHalfLog2e, b.y, b.z, b.w); s.c = make_float2(c.x, c.y); s.id = id;
            // fast-path eligibility (NaNs answer "generic"): alpha = opacity * G can exceed neither 0.99 nor, with
            // det >= 1e-5 trace^2 (smallest eigenvalue >= 1e-5 trace: ~100x the fp32 rounding of the three products),
            // can the computed power be positive
            const float A = a.z, B = a.w, Cc = b.x, tr = A + Cc;
            const bool fast = (b.y <= 0.99f) && (A > 0.f) && (Cc > 0.f) && (A * Cc - B * B > 1e-5f * tr * tr) &&
                              (fabsf(a.x) < 1e7f) && (fabsf(a.y) < 1e7f) && (tr < 1e7f);
            s.generic = fast ? 0u : 1u;
            sRec[j] = s;
            m = strip_mask<NH>(a, b, c.w, tx0, ty0);
        }
#pragma unroll
        for (int w = 0; w < NW; w++) {
            const uint32_t bits = __brev(__ballot_sync(0xffffffffu, (m >> w) & 1u));
            if (lane == 0 && (KB >= NT || wid < KB / 32)) sMask[w][wid + NW * h] = bits;     // word index = j / 32
        }
    }
}

#define GS_Q(v, q) (((q) & 1) ? (v)[(q) >> 1].y : (v)[(q) >> 1].x)

// The approximate evaluation shared by forward and backward: p = log2(e) * power, g = 2^p, a = opacity * g,
// d = a + nam (nam = -1/255 for a live pixel: sign-exact alpha >= 1/255 test; -inf for a dead one).  Returns true
// when one of the alphas sits inside the re-evaluation band around 1/255.
template <int NH>
__device__ __forceinline__ bool eval_alpha(const SRec& r, const float dx, const float2* dy, const float2* nam, float2* p,
                                           float2* g, float2* a, float2* d) {
    const float hA = (r.a.z * dx) * dx, hB = r.a.w * dx;
#pragma unroll
    for (int h = 0; h < NH; h++) {
        const float2 u = fma2(bc(r.b.x), dy[h], bc(hB));          // C2 dy + B2 dx
        p[h] = fma2(u, dy[h], bc(hA));                            // (C2 dy + B2 dx) dy + A2 dx dx
        g[h] = make_float2(ex2_approx(p[h].x), ex2_approx(p[h].y));
        a[h] = mul2(bc(r.b.y), g[h]);
        d[h] = add2(a[h], nam[h]);
    }
    float m = fminf(fabsf(d[0].x), fabsf(d[0].y));
    if (NH == 2) m = fminf(m, fminf(fabsf(d[NH - 1].x), fabsf(d[NH - 1].y)));
    return m < kBand;
}

// power and alpha (before the 0.99 clamp) of the thread's pixels with the reference's arithmetic (forward.cu:330-343),
// from the unscaled record
template <int NH>
__device__ __forceinline__ void exact_eval(const SRec& r, const float dx, const float2* dy,
                                           const float4* __restrict__ rec, float* power, float* alpha) {
    const float4 ra = __ldg(rec + (size_t)GS_REC_V4 * r.id), rb = __ldg(rec + (size_t)GS_REC_V4 * r.id + 1);
#pragma unroll
    for (int q = 0; q < 2 * NH; q++) {
        const float dyq = GS_Q(dy, q);
        power[q] = -0.5f * (ra.z * dx * dx + rb.x * dyq * dyq) - ra.w * dx * dyq;
        alpha[q] = r.b.y * expf(power[q]);
    }
}

}  // namespace
