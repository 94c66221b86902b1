// Tile compositing, forward and backward (sm_90a).
//
// k_blend_fwd replaces RAST/cuda_rasterizer/forward.cu:261-391 (renderCUDA): front-to-back alpha compositing of
//   colour + depth per 16x16 tile, same formulas per (pixel, splat).
// k_blend_bwd replaces backward.cu:399-586 (renderCUDA backward), same formulas per (pixel, splat).
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
//    of the four pixels are summed in registers, reduced across the warp with a value-halving shuffle butterfly
//    (12 shuffles for 9 values), written to a per-warp shared-memory slot with a plain store (each warp visits a
//    staged splat at most once), and leave the CTA as 128-bit vector reductions: one per (tile, splat).
//    1/(1-alpha) is a single MUFU.RCP (the gradient tolerance is 1e-3 relative).
// k_tile_partials (deterministic backward, opt-in) is k_blend_bwd with the reductions replaced by plain stores of the
//   same nine values per list position; gs_det_bwd.cu sums them per Gaussian in a fixed order.
// The default backward pass is gs_blend_bwd.cu (same arithmetic, a transposed shared-memory reduction instead of the
// shuffle butterfly, bit-identical sums); the kernels here stay selectable with GS_BLEND_BWD=0.
#include <cstdlib>

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

// Reduce 9 per-lane values across the warp with value halving: after step s every lane keeps only the half of
// the values selected by one bit of its lane id, so the 5 steps cost 5+3+2+1+1 = 12 shuffles (a plain
// butterfly needs 45).  On return even lanes whose (bit3,bit2,bit1) pattern is 000,001,010,100,101 hold in
// v[0] the full warp sum of value slot 5*bit4 + 3*bit3 + 2*bit2 + bit1; other lanes hold zeros/partials.
template <int N, int OFF>
__device__ __forceinline__ void halving_step(float* v, const int lane) {
    constexpr int Hh = (N + 1) / 2;
    const bool up = (lane & OFF) != 0;
#pragma unroll
    for (int k = 0; k < Hh; k++) {
        const float lo = v[k];
        const float hi = (k + Hh < N) ? v[k + Hh] : 0.f;
        const float send = up ? lo : hi;
        const float recv = __shfl_xor_sync(0xffffffffu, send, OFF);
        v[k] = (up ? hi : lo) + recv;
    }
}
__device__ __forceinline__ void warp_reduce9(float* v, const int lane) {
    halving_step<9, 16>(v, lane);
    halving_step<5, 8>(v, lane);
    halving_step<3, 4>(v, lane);
    halving_step<2, 2>(v, lane);
    halving_step<1, 1>(v, lane);
}

// The backward tile pass, shared by both flushes.  PARTS = false (k_blend_bwd): every (tile, splat) leaves the CTA as
// vector reductions into acc.  PARTS = true (k_tile_partials, the deterministic backward): the nine values of the pair
// at list position r (tile_off[tile] + pos) are STORED into part_a[2r], part_a[2r+1], part_b[r], and every pair of the
// tile that no pixel reached gets zeros, so all num_pairs entries are defined after the pass.
template <int NH, bool PARTS>
__device__ __forceinline__ void blend_bwd_tile(const GsView v, const uint32_t* __restrict__ tile_off,
                                               const uint32_t* __restrict__ list, const float4* __restrict__ rec,
                                               const float* __restrict__ final_Ts, const uint32_t* __restrict__ n_contrib,
                                               const float* __restrict__ dL_dpix, float4* __restrict__ acc,
                                               float4* __restrict__ part_a, float* __restrict__ part_b,
                                               const GsDevStatus* __restrict__ status, long long capacity) {
    constexpr int NW = Geo<NH>::NW, NT = Geo<NH>::NT, NQ = Geo<NH>::NQ;
    // a forward whose pair count exceeded the binning capacity rendered nothing (device-side guard): there is no list
    // to walk, the accumulators stay zero (static-capacity mode reports the overflow at the next host call)
    if ((long long)status->num_pairs > capacity) return;
    __shared__ SRec sRec[kBatch];
    __shared__ float sAcc[NW][kBatch * 9];               // per warp: plain stores, no atomics
    __shared__ uint32_t sMask[NW][kWords];
    __shared__ uint32_t sDone[NW][kWords];               // which slots of sAcc a warp has written this round
    __shared__ int sMax[NW];

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int tile = blockIdx.y * v.gx + blockIdx.x;
    const int tx0 = blockIdx.x * GS_TILE, ty0 = blockIdx.y * GS_TILE;
    const uint32_t px = tx0 + (lane & 15);
    const uint32_t pyb = ty0 + Geo<NH>::RW * wid + (lane >> 4);
    const float pixx = (float)px;
    float2 npy[NH];
#pragma unroll
    for (int h = 0; h < NH; h++) npy[h] = make_float2(-(float)(pyb + 4 * h), -(float)(pyb + 4 * h + 2));
    const uint32_t beg = tile_off[tile], end = tile_off[tile + 1];
    if (beg == end) return;

    const size_t HW = (size_t)v.H * v.W;
    const float bgc0 = __ldg(v.bg), bgc1 = __ldg(v.bg + 1), bgc2 = __ldg(v.bg + 2);
    BwdPix<NH> Q;
    int wmax = 0;
#pragma unroll
    for (int q = 0; q < NQ; q++) {
        const uint32_t py = pyb + 2 * q;
        const bool in = px < (uint32_t)v.W && py < (uint32_t)v.H;
        const uint32_t pix_id = (uint32_t)v.W * py + px;
        const float T_final = in ? final_Ts[pix_id] : 0.f;
        GS_Q(Q.T, q) = T_final;
        Q.last[q] = in ? (int)n_contrib[pix_id] : 0;
        const float g0 = in ? dL_dpix[pix_id] : 0.f, g1 = in ? dL_dpix[HW + pix_id] : 0.f, g2 = in ? dL_dpix[2 * HW + pix_id] : 0.f;
        GS_Q(Q.g0, q) = g0; GS_Q(Q.g1, q) = g1; GS_Q(Q.g2, q) = g2;
        float bd = 0.f;
        bd += bgc0 * g0; bd += bgc1 * g1; bd += bgc2 * g2;
        GS_Q(Q.tb, q) = -T_final * bd;
        GS_Q(Q.AR, q) = 0.f;
        wmax = max(wmax, Q.last[q]);
    }
    const float ddelx_dx = 0.5 * v.W, ddely_dy = 0.5 * v.H;

    // max of n_contrib over the warp's strip / over the tile: nothing behind it contributes
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) sMax[wid] = wmax;
    __syncthreads();
    int maxc = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) maxc = max(maxc, sMax[w]);
    if (PARTS) {                                         // behind every pixel's last contributor: zero partials
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (uint32_t r = beg + (uint32_t)maxc + tid; r < end; r += NT) {
            part_a[2 * (size_t)r] = z4; part_a[2 * (size_t)r + 1] = z4; part_b[r] = 0.f;
        }
    }

    // owner lanes / slots of the halving reduction
    const int b4 = (lane >> 4) & 1, b3 = (lane >> 3) & 1, b2 = (lane >> 2) & 1, b1 = (lane >> 1) & 1;
    const int slot = 5 * b4 + 3 * b3 + 2 * b2 + b1;
    const bool owner = ((lane & 1) == 0) && !(b3 && b2) && !(b3 == 0 && b2 && b1) && slot < 9;
    float* const myAcc = sAcc[wid] + (owner ? slot : 0);

    for (int hi = maxc; hi > 0; hi -= kBatch) {
        __syncthreads();
        const int cnt = min(kBatch, hi);
        // slot j holds list position hi-1-j: reverse traversal = increasing j
        stage_batch<NH, kBatch>(sRec, sMask, list, rec, beg, cnt, tx0, ty0, [&](int j) { return hi - 1 - j; });
        __syncthreads();
#pragma unroll 1
        for (int k = 0; k < kWords; k++) {
            uint32_t bits = sMask[wid][k];
            uint32_t done = 0;
            while (bits) {
                const int lz = __clz(bits);
                const uint32_t bit = 0x80000000u >> lz;
                bits &= ~bit;
                const int j = 32 * k + lz;
                const int pos = hi - 1 - j;      // 0-based list position
                if (pos >= wmax) continue;       // behind every pixel of this strip
                const SRec& r = sRec[j];
                const float dx = r.a.x - pixx;
                float2 dy[NH], p[NH], g[NH], a[NH], d[NH];
#pragma unroll
                for (int h = 0; h < NH; h++) dy[h] = add2(bc(r.a.y), npy[h]);
                float2 nam[NH];
#pragma unroll
                for (int h = 0; h < NH; h++) nam[h] = bc(-kAlphaMin);
                const bool band = eval_alpha<NH>(r, dx, dy, nam, p, g, a, d);
                float vv[9];
                bool any;
                if (band || r.generic) {
#pragma unroll
                    for (int q = 0; q < 9; q++) vv[q] = 0.f;
                    any = bwd_generic<NH>(Q, r, dx, dy, p, g, a, band, pos, rec, vv);
                } else {
                    // fast path: alpha = a (no clamp), contributes <=> pos < last && d >= 0; a skipped pixel runs with
                    // alpha = 0, which makes every update a no-op (T / 1 = T, AR + 0, zero weights)
                    float2 ae[NH];
#pragma unroll
                    for (int q = 0; q < NQ; q++) GS_Q(ae, q) = (pos < Q.last[q] && GS_Q(d, q) >= 0.f) ? GS_Q(a, q) : 0.f;
                    uint32_t anyb = __float_as_uint(ae[0].x) | __float_as_uint(ae[0].y);
                    if (NH == 2) anyb |= __float_as_uint(ae[NH - 1].x) | __float_as_uint(ae[NH - 1].y);
                    any = anyb != 0u;
                    float2 c0 = bc(0.f), c1 = bc(0.f), c2 = bc(0.f), s0 = bc(0.f), sy = bc(0.f), syy = bc(0.f);
#pragma unroll
                    for (int h = 0; h < NH; h++) {
                        const float2 om = fma2(ae[h], bc(-1.f), bc(1.f));                     // 1 - alpha
                        const float2 inv = make_float2(rcp_approx(om.x), rcp_approx(om.y));
                        Q.T[h] = mul2(Q.T[h], inv);                                           // T of the splats in front
                        const float2 cg = fma2(bc(r.c.x), Q.g2[h], fma2(bc(r.b.w), Q.g1[h], mul2(bc(r.b.z), Q.g0[h])));
                        const float2 dcol = fma2(Q.AR[h], bc(-1.f), cg);                      // cg - AR
                        Q.AR[h] = fma2(ae[h], dcol, Q.AR[h]);
                        const float2 dch = mul2(ae[h], Q.T[h]);                               // dchannel_dcolor
                        c0 = fma2(dch, Q.g0[h], c0); c1 = fma2(dch, Q.g1[h], c1); c2 = fma2(dch, Q.g2[h], c2);
                        const float2 dLda = fma2(dcol, Q.T[h], mul2(Q.tb[h], inv));           // dL_dalpha
                        const float2 wq = mul2(ae[h], dLda);                                  // opacity G dL_dalpha
                        s0 = add2(s0, wq);
                        const float2 t = mul2(wq, dy[h]);
                        sy = add2(sy, t);
                        syy = fma2(t, dy[h], syy);
                    }
                    vv[0] = c0.x + c0.y; vv[1] = c1.x + c1.y; vv[2] = c2.x + c2.y;
                    const float S0 = s0.x + s0.y, SY = sy.x + sy.y;
                    vv[3] = S0; vv[4] = dx * S0; vv[5] = SY;
                    vv[6] = dx * vv[4]; vv[7] = dx * SY; vv[8] = syy.x + syy.y;
                }
                if (!__any_sync(0xffffffffu, any)) continue;
                warp_reduce9(vv, lane);
                if (owner) myAcc[j * 9] = vv[0];
                done |= bit;
            }
            if (lane == 0) sDone[wid][k] = done;
        }
        __syncthreads();
#pragma unroll
        for (int h = 0; h < kBatch / NT; h++) {
            const int j = tid + h * NT;
            if (j < cnt) {
                const uint32_t bit = 0x80000000u >> (j & 31);
                bool dn[NW];
                bool anyd = false;
#pragma unroll
                for (int w = 0; w < NW; w++) { dn[w] = (sDone[w][j >> 5] & bit) != 0u; anyd = anyd || dn[w]; }
                float4 f0 = make_float4(0.f, 0.f, 0.f, 0.f), f1 = f0;
                float f2 = 0.f;
                if (anyd) {
                    float r[9];
#pragma unroll
                    for (int k = 0; k < 9; k++) {
                        float x = 0.f;
#pragma unroll
                        for (int w = 0; w < NW; w++) x += dn[w] ? sAcc[w][j * 9 + k] : 0.f;
                        r[k] = x;
                    }
                    flush_values(sRec[j], r, ddelx_dx, ddely_dy, f0, f1, f2);
                    if (!PARTS) {
                        float4* dst = acc + (size_t)3 * sRec[j].id;
                        atomicAdd(dst, f0);
                        atomicAdd(dst + 1, f1);
                        atomicAdd(reinterpret_cast<float*>(dst + 2), f2);
                    }
                }
                if (PARTS) {
                    const size_t pr = (size_t)beg + (size_t)(hi - 1 - j);
                    part_a[2 * pr] = f0; part_a[2 * pr + 1] = f1; part_b[pr] = f2;
                }
            }
        }
    }
}

template <int NH, int OCC>
__global__ void __launch_bounds__(Geo<NH>::NT, OCC)
k_blend_bwd(const GsView v, const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ list,
            const float4* __restrict__ rec, const float* __restrict__ final_Ts,
            const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpix, float4* __restrict__ acc,
            const GsDevStatus* __restrict__ status, long long capacity) {
    blend_bwd_tile<NH, false>(v, tile_off, list, rec, final_Ts, n_contrib, dL_dpix, acc, nullptr, nullptr, status, capacity);
}

// Deterministic backward, tile pass: k_blend_bwd's traversal and arithmetic, partials stored per list position
template <int NH, int OCC>
__global__ void __launch_bounds__(Geo<NH>::NT, OCC)
k_tile_partials(const GsView v, const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ list,
                const float4* __restrict__ rec, const float* __restrict__ final_Ts,
                const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpix, float4* __restrict__ part_a,
                float* __restrict__ part_b, const GsDevStatus* __restrict__ status, long long capacity) {
    blend_bwd_tile<NH, true>(v, tile_off, list, rec, final_Ts, n_contrib, dL_dpix, nullptr, part_a, part_b, status, capacity);
}

}  // namespace

int g_gs_blend_variant = 0;           // GS_BLEND_VARIANT=2 / 3 force the 16x8 / 16x4 warp geometry (A/B measurements)
int g_gs_num_sms = 132;           // H100 SXM; replaced by the device's count when a context is created

// 16x4 strips (4 warps per tile) when 16x8 blocks would leave the SMs with fewer than ~20 resident warps
bool gs_blend_use_strips(const GsView& v) {
    if (g_gs_blend_variant == 2) return false;
    if (g_gs_blend_variant == 3) return true;
    return (long long)v.gx * v.gy * 2 < (long long)g_gs_num_sms * 20;
}

void gs_launch_blend_fwd(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                         const GsDevStatus* status, long long capacity, float* final_T, uint32_t* n_contrib,
                         float* out_color, float* out_depth, cudaStream_t s) {
    dim3 grid(v.gx, v.gy);
    // CTAs per SM the register allocation aims at: 14 (72 registers, 28 warps per SM); 12 (80 registers) measured the same
    // on config 3 (H100 SXM, 400 W limit: 0.127 vs 0.128 ms); GS_BLEND_OCC_FWD=12 keeps the other build for A/B runs
    static const int occ = getenv("GS_BLEND_OCC_FWD") ? atoi(getenv("GS_BLEND_OCC_FWD")) : 14;
    if (gs_blend_use_strips(v))
        k_blend_fwd<1, 6><<<grid, Geo<1>::NT, 0, s>>>(v, tile_off, list, rec, status, capacity, final_T, n_contrib, out_color, out_depth);
    else if (occ == 12)
        k_blend_fwd<2, 12><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, status, capacity, final_T, n_contrib, out_color, out_depth);
    else
        k_blend_fwd<2, 14><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, status, capacity, final_T, n_contrib, out_color, out_depth);
}
void gs_launch_blend_bwd_shfl(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                              const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, float4* acc,
                              const GsDevStatus* status, long long capacity, cudaStream_t s) {
    dim3 grid(v.gx, v.gy);
    // 13 CTAs per SM (72 registers, 4 bytes spilled; shared memory then limits at 13): 0.258 ms against 0.267-0.275 ms
    // for 10 (88 registers) on config 3 (H100 SXM, 400 W limit)
    static const int occ = getenv("GS_BLEND_OCC_BWD") ? atoi(getenv("GS_BLEND_OCC_BWD")) : 13;
    if (gs_blend_use_strips(v))
        k_blend_bwd<1, 7><<<grid, Geo<1>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, acc, status, capacity);
    else if (occ == 10)
        k_blend_bwd<2, 10><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, acc, status, capacity);
    else
        k_blend_bwd<2, 13><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, acc, status, capacity);
}
void gs_launch_tile_partials_shfl(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                                  const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, float4* part_a,
                                  float* part_b, const GsDevStatus* status, long long capacity, cudaStream_t s) {
    dim3 grid(v.gx, v.gy);
    // same geometry choice and register targets as gs_launch_blend_bwd_shfl
    if (gs_blend_use_strips(v))
        k_tile_partials<1, 7><<<grid, Geo<1>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, part_a, part_b,
                                                          status, capacity);
    else
        k_tile_partials<2, 13><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, part_a, part_b,
                                                           status, capacity);
}
