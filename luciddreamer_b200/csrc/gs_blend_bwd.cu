// Backward tile pass (sm_90a): k_blend_bwd and k_tile_partials, the reverse traversal of gs_blend.cu's forward.
//
// Staging, the alpha evaluation and the skip decision are the forward's (gs_blend.cuh).  Per hit splat every lane
// computes nine values vv[0..8] for its pixels (BwdPix), and the per-(tile, splat) sums are formed as follows:
//  * each warp buffers the lanes' values of kGroup = 3 hit splats in its own slab, [splat][value][lane] (27 rows of
//    32 lanes, rows padded to 36 words): 9 plain STS per splat, conflict-free;
//  * when the slab is full (or the batch ends), lane i < 27 sums row i: 8 LDS.128 (8 consecutive lanes read 8
//    distinct 4-bank groups thanks to the padding) and 31 FADD in a fixed tree order -- pairs (l, l^16) first, then
//    the partials 8, 4, 2, 1 apart (slab_row_sum);
//  * the sum goes to the warp's per-splat slot in shared memory, and the CTA sums the warps and flushes the sums
//    (flush_values, then red.global.add.v4.f32 or the stores of the deterministic partials).
// That tree order is the deterministic backward's contract: k_tile_partials stores its sums, and gs_det_bwd.cu adds
// them in a fixed order, so changing the tree changes the deterministic gradients' bits.
// The slab costs 3.9 KB per warp; the batch is 64 splats (config 3 has ~49 pairs per tile after exact culling), which
// keeps shared memory per CTA at 15 KB (NH = 2).

#include "gs_blend.cuh"

namespace {

constexpr int kBatch = 64;            // splats staged per round
constexpr int kWords = kBatch / 32;
constexpr int kGroup = 3;             // hit splats per slab: 27 (splat, value) rows, one per lane
constexpr int kRows = 9 * kGroup;
constexpr int kStride = 36;           // slab row: 32 lanes + 4 words of padding (16-byte aligned rows)

constexpr float kUnscale = -2.0f * 0.6931471805599453f;   // undoes stage_batch's conic scaling for the flush

template <int NH> struct BwdPix {
    float2 T[NH];
    float2 tb[NH];                    // -T_final * (bg . dL_dpixel)
    float2 AR[NH];                    // sum_ch accum_rec_ch * dL_dpixel_ch, already advanced past the last contributing splat
    float2 g0[NH], g1[NH], g2[NH];    // dL_dpixel
    int last[2 * NH];                 // last contributor (1-based list position)
};

// What both backward paths sum per (thread, splat), for w = opacity * G * dL_dalpha of the contributing pixels:
//   vv[0..2] = sum alpha T dL_dpixel_ch          (dL_dcolor)
//   vv[3..8] = sum w, dx w, sum w dy, dx dx w, dx sum w dy, sum w dy dy
// backward.cu:563-583 needs G dL_dalpha times {1, dx, dy, dx dx, dx dy, dy dy} and the splat's constants (A, B, C,
// -0.5 W, -0.5 H, -0.5, 1/opacity), which are applied once per (tile, splat) at the flush.
//
// backward.cu:520-528 keeps accum_rec per channel and forms sum_ch (c_ch - accum_rec_ch) * dL_dpixel_ch.  dL_dpixel is
// constant per pixel, so only the scalar AR = sum_ch accum_rec_ch * dL_dpixel_ch is carried: it obeys the same
// recurrence (AR' = a cg + (1 - a) AR = AR + a (cg - AR), cg = c . dL_dpixel) and is advanced eagerly.

// generic path of the backward: the reference's test sequence per pixel, exact alpha inside the band
template <int NH>
__device__ __forceinline__ bool bwd_generic(BwdPix<NH>& Q, const SRec& r, const float dx, const float2* dy, const float2* p,
                                            const float2* g, const float2* a, const bool band, const int pos,
                                            const float4* __restrict__ rec, float* vv) {
    (void)g;
    float alpha[2 * NH], power[2 * NH];          // alpha = opacity * G, unclamped
#pragma unroll
    for (int q = 0; q < 2 * NH; q++) { alpha[q] = GS_Q(a, q); power[q] = GS_Q(p, q); }
    if (band || r.generic) exact_eval<NH>(r, dx, dy, rec, power, alpha);
    bool any = false;
    float s0 = 0.f, sy = 0.f, syy = 0.f;
#pragma unroll
    for (int q = 0; q < 2 * NH; q++) {
        const float al = fminf(0.99f, alpha[q]);
        const bool ok = (pos < Q.last[q]) && !(power[q] > 0.0f) && !(al < kAlphaMin);
        any = any || ok;
        const float a_ = ok ? al : 0.f;                     // alpha = 0 makes every update below a no-op
        const float inv = rcp_approx(1.f - a_);
        float& T = GS_Q(Q.T, q);
        T = T * inv;
        const float g0 = GS_Q(Q.g0, q), g1 = GS_Q(Q.g1, q), g2 = GS_Q(Q.g2, q);
        const float cg = fmaf(r.c.x, g2, fmaf(r.b.w, g1, r.b.z * g0));
        float& AR = GS_Q(Q.AR, q);
        const float dcol = cg - AR;
        AR = fmaf(a_, dcol, AR);
        const float dch = a_ * T;
        vv[0] = fmaf(dch, g0, vv[0]); vv[1] = fmaf(dch, g1, vv[1]); vv[2] = fmaf(dch, g2, vv[2]);
        const float dL_dalpha = fmaf(dcol, T, GS_Q(Q.tb, q) * inv);
        const float oG = ok ? alpha[q] : 0.f;               // opacity * G; zero keeps an inf of a skipped splat out of the sums
        const float wq = oG * dL_dalpha;
        const float dyq = GS_Q(dy, q);
        s0 += wq;
        const float t = wq * dyq;
        sy += t;
        syy = fmaf(t, dyq, syy);
    }
    vv[3] = s0;  vv[4] = dx * s0;  vv[5] = sy;
    vv[6] = dx * vv[4];  vv[7] = dx * sy;  vv[8] = syy;
    return any;
}

// The nine values one (tile, splat) contributes to the splat's accumulator, from the tile sums r[0..8] (see
// BwdPix): what k_blend_bwd adds into acc and what k_tile_partials stores.  Both kernels run this one expression.
__device__ __forceinline__ void flush_values(const SRec& sr, const float* r, const float ddelx_dx, const float ddely_dy,
                                             float4& f0, float4& f1, float& f2) {
    // r[3..8] = sums of w, w dx, w dy, w dx dx, w dx dy, w dy dy (w = opacity G dL_dalpha) over the tile
    const float A = sr.a.z * kUnscale, B = sr.a.w * (0.5f * kUnscale), C = sr.b.x * kUnscale;
    const float kx = r[4], ky = r[5], hf = -0.5f;
    f0 = make_float4(-(A * kx + B * ky) * ddelx_dx, -(C * ky + B * kx) * ddely_dy, hf * r[6], hf * r[7]);
    f1 = make_float4(hf * r[8], r[3] * rcp_approx(sr.b.y), r[0], r[1]);
    f2 = r[2];
}

// The slab and the staged records are read and written through 32-bit shared-window addresses (ld/st.shared): the
// slab's stores and loads stay in the order the __syncwarp()s give them, and the record's fields are plain loads the
// compiler schedules as it likes (measured on config 3: 2 % off k_blend_bwd against reading the record through a
// reference into sRec).
__device__ __forceinline__ void sts(const uint32_t addr, const float x) {
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(x) : "memory");
}
__device__ __forceinline__ float4 lds4(const uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
// a staged record: loads the compiler may move or drop (the records do not change between the barriers, and the
// address depends on the mask word read after the barrier)
__device__ __forceinline__ float4 lds4_rec(const uint32_t addr) {
    float4 v;
    asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_rec(const uint32_t addr) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ SRec load_srec(const uint32_t addr) {
    SRec r;
    r.a = lds4_rec(addr);
    r.b = lds4_rec(addr + 16);
    r.c = make_float2(__uint_as_float(lds_rec(addr + 32)), __uint_as_float(lds_rec(addr + 36)));
    r.id = lds_rec(addr + 40);
    r.generic = lds_rec(addr + 44);
    return r;
}

// Lane i < 9 * n sums slab row i over the 32 lanes: element l is first added to element l + 16, then the partials to the
// one 8, 4, 2, 1 further.  The deterministic backward's gradients depend on this order bit for bit.
__device__ __forceinline__ float slab_row_sum(const uint32_t row) {
    float4 s1[4];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const float4 lo = lds4(row + 16 * c), hi = lds4(row + 16 * (c + 4));     // elements 4c.. and 4c+16..
        s1[c] = make_float4(lo.x + hi.x, lo.y + hi.y, lo.z + hi.z, lo.w + hi.w);
    }
    float4 s2[2];
#pragma unroll
    for (int c = 0; c < 2; c++)
        s2[c] = make_float4(s1[c].x + s1[c + 2].x, s1[c].y + s1[c + 2].y, s1[c].z + s1[c + 2].z, s1[c].w + s1[c + 2].w);
    const float4 s3 = make_float4(s2[0].x + s2[1].x, s2[0].y + s2[1].y, s2[0].z + s2[1].z, s2[0].w + s2[1].w);
    return (s3.x + s3.z) + (s3.y + s3.w);
}

// The backward tile pass, shared by both flushes.  PARTS = false (k_blend_bwd): every (tile, splat) leaves the CTA as
// vector reductions into acc.  PARTS = true (k_tile_partials, the deterministic backward): the nine values of the pair
// at list position r (tile_off[tile] + pos) are STORED into part_a[2r], part_a[2r+1], part_b[r], and every pair of the
// tile that no pixel reached gets zeros, so all num_pairs entries are defined after the pass.
template <int NH, bool PARTS>
__device__ __forceinline__ void blend_bwd_tile_slab(const GsView v, const uint32_t* __restrict__ tile_off,
                                                    const uint32_t* __restrict__ list, const float4* __restrict__ rec,
                                                    const float* __restrict__ final_Ts,
                                                    const uint32_t* __restrict__ n_contrib,
                                                    const float* __restrict__ dL_dpix, float4* __restrict__ acc,
                                                    float4* __restrict__ part_a, float* __restrict__ part_b,
                                                    const GsDevStatus* __restrict__ status, long long capacity) {
    constexpr int NW = Geo<NH>::NW, NT = Geo<NH>::NT, NQ = Geo<NH>::NQ;
    constexpr int NR = (kBatch + NT - 1) / NT;
    if ((long long)status->num_pairs > capacity) return;
    __shared__ SRec sRec[kBatch];
    __shared__ float sAcc[NW][kBatch * 9];               // per warp: the warp's nine sums per staged splat
    __shared__ __align__(16) float sSlab[NW][kRows * kStride];
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

    static_assert(sizeof(SRec) == 48, "load_srec reads the record by offsets");
    const uint32_t srec = (uint32_t)__cvta_generic_to_shared(sRec);
    const uint32_t slab = (uint32_t)__cvta_generic_to_shared(sSlab[wid]);
    const uint32_t slab_col = slab + 4 * lane;           // this lane's column: its values of every buffered splat
    const uint32_t slab_row = slab + 4 * kStride * lane; // the row this lane sums (lane < kRows)
    float* const acc_warp = sAcc[wid];
    const int own_g = lane / 9, own_k = lane - 9 * own_g;          // (buffered splat, value) of the row
    int ng = 0;                                          // splats in the slab
    int own_j = 0;                                       // batch slot of splat own_g
    auto reduce_slab = [&]() {
        __syncwarp();
        if (lane < 9 * ng) acc_warp[own_j * 9 + own_k] = slab_row_sum(slab_row);
        __syncwarp();                                    // the rows are read before the next splat overwrites them
        ng = 0;
    };

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
                const SRec r = load_srec(srec + (uint32_t)j * (uint32_t)sizeof(SRec));
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
                    // the sums start from the first pair's terms: x + 0 == x, except that a -0 term stays -0, which
                    // only the sign of a zero sum can show and no output does
                    float2 c0, c1, c2, s0, sy, syy;
#pragma unroll
                    for (int h = 0; h < NH; h++) {
                        const float2 om = fma2(ae[h], bc(-1.f), bc(1.f));                     // 1 - alpha
                        const float2 inv = make_float2(rcp_approx(om.x), rcp_approx(om.y));
                        Q.T[h] = mul2(Q.T[h], inv);                                           // T of the splats in front
                        const float2 cg = fma2(bc(r.c.x), Q.g2[h], fma2(bc(r.b.w), Q.g1[h], mul2(bc(r.b.z), Q.g0[h])));
                        const float2 dcol = fma2(Q.AR[h], bc(-1.f), cg);                      // cg - AR
                        Q.AR[h] = fma2(ae[h], dcol, Q.AR[h]);
                        const float2 dch = mul2(ae[h], Q.T[h]);                               // dchannel_dcolor
                        const float2 dLda = fma2(dcol, Q.T[h], mul2(Q.tb[h], inv));           // dL_dalpha
                        const float2 wq = mul2(ae[h], dLda);                                  // opacity G dL_dalpha
                        const float2 t = mul2(wq, dy[h]);
                        if (h == 0) {
                            c0 = mul2(dch, Q.g0[h]); c1 = mul2(dch, Q.g1[h]); c2 = mul2(dch, Q.g2[h]);
                            s0 = wq; sy = t; syy = mul2(t, dy[h]);
                        } else {
                            c0 = fma2(dch, Q.g0[h], c0); c1 = fma2(dch, Q.g1[h], c1); c2 = fma2(dch, Q.g2[h], c2);
                            s0 = add2(s0, wq); sy = add2(sy, t); syy = fma2(t, dy[h], syy);
                        }
                    }
                    vv[0] = c0.x + c0.y; vv[1] = c1.x + c1.y; vv[2] = c2.x + c2.y;
                    const float S0 = s0.x + s0.y, SY = sy.x + sy.y;
                    vv[3] = S0; vv[4] = dx * S0; vv[5] = SY;
                    vv[6] = dx * vv[4]; vv[7] = dx * SY; vv[8] = syy.x + syy.y;
                }
                if (!__any_sync(0xffffffffu, any)) continue;
                const uint32_t col = slab_col + ng * (4 * 9 * kStride);
#pragma unroll
                for (int q = 0; q < 9; q++) sts(col + 4 * kStride * q, vv[q]);
                own_j = (own_g == ng) ? j : own_j;
                done |= bit;
                if (++ng == kGroup) reduce_slab();
            }
            if (lane == 0) sDone[wid][k] = done;
        }
        if (ng) reduce_slab();
        __syncthreads();
#pragma unroll
        for (int h = 0; h < NR; h++) {
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
    blend_bwd_tile_slab<NH, false>(v, tile_off, list, rec, final_Ts, n_contrib, dL_dpix, acc, nullptr, nullptr, status,
                                   capacity);
}

// Deterministic backward, tile pass: k_blend_bwd's traversal and arithmetic, partials stored per list position
template <int NH, int OCC>
__global__ void __launch_bounds__(Geo<NH>::NT, OCC)
k_tile_partials(const GsView v, const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ list,
                const float4* __restrict__ rec, const float* __restrict__ final_Ts,
                const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpix, float4* __restrict__ part_a,
                float* __restrict__ part_b, const GsDevStatus* __restrict__ status, long long capacity) {
    blend_bwd_tile_slab<NH, true>(v, tile_off, list, rec, final_Ts, n_contrib, dL_dpix, nullptr, part_a, part_b, status,
                                  capacity);
}

}  // namespace

// Register targets: 13 CTAs per SM for 16x8 blocks, 7 for 16x4 strips
void gs_launch_blend_bwd(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                         const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, float4* acc,
                         const GsDevStatus* status, long long capacity, cudaStream_t s) {
    dim3 grid(v.gx, v.gy);
    if (gs_blend_use_strips(v))
        k_blend_bwd<1, 7><<<grid, Geo<1>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, acc, status, capacity);
    else
        k_blend_bwd<2, 13><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, acc, status, capacity);
}
void gs_launch_tile_partials(const GsView& v, const uint32_t* tile_off, const uint32_t* list, const float4* rec,
                             const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, float4* part_a,
                             float* part_b, const GsDevStatus* status, long long capacity, cudaStream_t s) {
    dim3 grid(v.gx, v.gy);
    if (gs_blend_use_strips(v))
        k_tile_partials<1, 7><<<grid, Geo<1>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, part_a, part_b,
                                                          status, capacity);
    else
        k_tile_partials<2, 13><<<grid, Geo<2>::NT, 0, s>>>(v, tile_off, list, rec, final_T, n_contrib, dL_dpix, part_a, part_b,
                                                           status, capacity);
}
