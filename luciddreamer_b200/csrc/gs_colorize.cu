// Depth colour mapping for the video path (sm_90a): the step render_video runs after its loop
// (luciddreamer.py:267, `depthlist = [colorize(depth) for depth in depthlist]`, utils/depth.py:7-62), for a whole clip.
//
// Per frame, over the valid pixels (value != invalid_val):
//   vmin = np.percentile(valid, 2), vmax = np.percentile(valid, 98)      -- numpy's float32 arithmetic, restated below
//   x = (value - vmin) / (vmax - vmin) if vmin != vmax else value * 0     -- IEEE float32 sub / div
//   rgba = lut[clamp(trunc(x * 256), 0, 255)] (x < 0 -> 0, x > 1 -> 255), background for invalid pixels
//
// The four order statistics the two percentiles need are found by an exact radix select over an ordered 32-bit key
// (11 + 11 + 10 bits), for every frame of the batch in one fixed sequence of launches: no host loop, no host sync, no
// float atomics.  Histograms are built in shared memory per CTA and merged with integer atomics, so every result is
// independent of scheduling.
//
//   k_cz_hist<1>    histogram of key[31:21] per frame (its total is the frame's valid-pixel count n)
//   k_cz_select<1>  n -> the ranks of the 2nd / 98th percentiles (<= 4 order statistics) -> their 11-bit buckets
//   k_cz_hist<2>    histogram of key[20:10] over the pixels whose key[31:21] is one of the selected buckets
//   k_cz_select<2>
//   k_cz_hist<3>    histogram of key[9:0] over the pixels whose key[31:10] is one of the selected 22-bit prefixes
//   k_cz_select<3>  exact keys -> values -> numpy's float32 _lerp -> vmin / vmax per frame
//   k_cz_color      one RGBA word per pixel (128-bit loads and stores per 4 pixels where the frame is aligned)
#include <cstddef>

#include "gs_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTargets = 4;                       // order statistics per frame: floor / ceil of each percentile's index
constexpr int kBins12 = 2048;                     // passes 1 and 2: 11 bits
constexpr int kBins3 = 1024;                      // pass 3: 10 bits
constexpr size_t kOff2 = kBins12;                 // per-frame word offsets of the three histograms
constexpr size_t kOff3 = kOff2 + (size_t)kTargets * kBins12;
constexpr size_t kFrameWords = kOff3 + (size_t)kTargets * kBins3;
constexpr int kGroupsPerThreadHist = 16;          // 64 pixels per thread between shared-histogram clears / flushes
constexpr int kGroupsPerThreadColor = 4;
constexpr uint32_t kNoPrefix = 0xffffffffu;       // never equals a key prefix of 11 or 22 bits
static_assert(kThreads == 256, "k_cz_color loads the 256-entry table with one word per thread");

// Per-frame selection state, written by k_cz_select<PASS> and read by the next pass.
struct CzState {
    uint32_t n;                   // valid pixels
    uint32_t nslots;              // distinct prefixes the next histogram pass counts (0: nothing to select)
    uint32_t prefix[kTargets];    // slot -> key prefix (kNoPrefix when unused)
    uint32_t slot[kTargets];      // target -> slot
    uint32_t rank[kTargets];      // target -> rank among the pixels that share its prefix
    float vmin, vmax;             // after pass 3
};
static_assert(sizeof(CzState) == 64, "CzState is 16 words");

// Ordered key: unsigned order == float order, and -0.0 / +0.0 share one key (numpy's partition treats them as equal).
__device__ __forceinline__ uint32_t cz_key(float f) {
    uint32_t b = __float_as_uint(f);
    if ((b << 1) == 0u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float cz_unkey(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Up to 4 consecutive pixels p..p+3 of one frame; cnt = how many exist.
__device__ __forceinline__ int cz_load4(const float* __restrict__ v, long long HW, long long p, bool vec, float x[4]) {
    if (p >= HW) return 0;
    if (vec && p + 3 < HW) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(v + p));
        x[0] = q.x; x[1] = q.y; x[2] = q.z; x[3] = q.w;
        return 4;
    }
    const int cnt = (int)min(4LL, HW - p);
#pragma unroll
    for (int k = 0; k < 4; k++) x[k] = k < cnt ? v[p + k] : 0.f;
    return cnt;
}

// Shared-histogram increment called by all 32 lanes; bin < 0 = nothing to count.  A warp whose lanes all hit one bin
// (background, tied depths) adds once.
__device__ __forceinline__ void cz_warp_add(uint32_t* sh, int bin) {
    const int lead = __shfl_sync(0xffffffffu, bin, 0);
    if (__all_sync(0xffffffffu, bin == lead)) {
        if ((threadIdx.x & 31) == 0 && lead >= 0) atomicAdd(&sh[lead], 32u);
    } else if (bin >= 0) {
        atomicAdd(&sh[bin], 1u);
    }
}

template <int PASS>
__global__ void __launch_bounds__(kThreads)
k_cz_hist(const float* __restrict__ value, const long long HW, const int F, const float invalid_val,
          uint32_t* __restrict__ bins, const CzState* __restrict__ st) {
    constexpr int NB = PASS == 3 ? kBins3 : kBins12;
    constexpr int NS = PASS == 1 ? 1 : kTargets;
    constexpr size_t OFF = PASS == 1 ? 0 : PASS == 2 ? kOff2 : kOff3;
    __shared__ uint32_t sh[NS * NB];
    const long long groups = (HW + 3) >> 2;
    for (int f = blockIdx.y; f < F; f += gridDim.y) {
        int ns = 1;
        uint32_t pref[kTargets];
#pragma unroll
        for (int j = 0; j < kTargets; j++) pref[j] = kNoPrefix;
        if (PASS > 1) {
            ns = (int)st[f].nslots;                         // uniform over the CTA
            if (ns == 0) continue;
#pragma unroll
            for (int j = 0; j < kTargets; j++) pref[j] = st[f].prefix[j];
        }
        for (int i = threadIdx.x; i < ns * NB; i += kThreads) sh[i] = 0u;
        __syncthreads();
        const float* v = value + (size_t)f * (size_t)HW;
        const bool vec = (reinterpret_cast<uintptr_t>(v) & 15) == 0;
        // every thread of the CTA runs the same number of iterations (the warp-wide votes in cz_warp_add need that)
        for (long long g0 = (long long)blockIdx.x * kThreads; g0 < groups; g0 += (long long)gridDim.x * kThreads) {
            float x[4];
            const int cnt = cz_load4(v, HW, (g0 + threadIdx.x) * 4, vec, x);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                int bin = -1;
                if (k < cnt && x[k] != invalid_val) {
                    const uint32_t key = cz_key(x[k]);
                    if (PASS == 1) {
                        bin = (int)(key >> 21);
                    } else {
                        const uint32_t hi = PASS == 2 ? key >> 21 : key >> 10;
                        const int digit = PASS == 2 ? (int)((key >> 10) & 2047u) : (int)(key & 1023u);
#pragma unroll
                        for (int j = 0; j < kTargets; j++)
                            if (hi == pref[j]) bin = j * NB + digit;
                    }
                }
                cz_warp_add(sh, bin);
            }
        }
        __syncthreads();
        uint32_t* gb = bins + (size_t)f * kFrameWords + OFF;
        for (int i = threadIdx.x; i < ns * NB; i += kThreads) {
            const uint32_t c = sh[i];
            if (c) atomicAdd(&gb[i], c);
        }
        __syncthreads();
    }
}

// numpy's percentile index for float32 data (method "linear"): q = float32(p) / float32(100), index = (n - 1) * q in
// float32; floor / floor + 1 are the two order statistics, gamma = index - floor.  At or past the last element both
// are the last element and numpy's gamma is index - (-1).
__device__ __forceinline__ void cz_index(uint32_t n, float p, uint32_t& lo, uint32_t& hi, float& gamma) {
    const float q = __fdiv_rn(p, 100.f);
    const float last = __uint2float_rn(n - 1u);
    const float v = __fmul_rn(last, q);
    if (v >= last) {
        lo = hi = n - 1u;
        gamma = __fadd_rn(v, 1.f);
    } else {
        const float fl = floorf(v);
        lo = (uint32_t)fl;
        hi = lo + 1u;
        gamma = __fsub_rn(v, fl);
    }
}

// numpy's _lerp: a + (b - a) * t, or b - (b - a) * (1 - t) where t >= 0.5; float32, no contraction.
__device__ __forceinline__ float cz_lerp(float a, float b, float t) {
    const float d = __fsub_rn(b, a);
    return t >= 0.5f ? __fsub_rn(b, __fmul_rn(d, __fsub_rn(1.f, t))) : __fadd_rn(a, __fmul_rn(d, t));
}

// One CTA per frame: for every target, find the bucket of the pass-PASS histogram that holds its rank.
template <int PASS>
__global__ void __launch_bounds__(kThreads)
k_cz_select(uint32_t* __restrict__ bins, CzState* __restrict__ st, float* __restrict__ vminmax) {
    constexpr int NB = PASS == 3 ? kBins3 : kBins12;
    constexpr int PER = NB / kThreads;
    constexpr size_t OFF = PASS == 1 ? 0 : PASS == 2 ? kOff2 : kOff3;
    __shared__ uint32_t s_warp[kThreads / 32];
    __shared__ uint32_t s_rank[kTargets], s_slot[kTargets], s_bin[kTargets], s_res[kTargets];
    __shared__ uint32_t s_ns, s_n;
    const int f = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    CzState& S = st[f];
    if (threadIdx.x == 0) {
        s_ns = PASS == 1 ? 1u : S.nslots;
#pragma unroll
        for (int t = 0; t < kTargets; t++) {
            s_slot[t] = PASS == 1 ? 0u : S.slot[t];
            s_rank[t] = PASS == 1 ? 0u : S.rank[t];
        }
    }
    __syncthreads();
    const int ns = (int)s_ns;
    if (ns == 0) return;                                   // frame without valid pixels: its state stays as pass 1 left it
    for (int j = 0; j < ns; j++) {
        const uint32_t* h = bins + (size_t)f * kFrameWords + OFF + (size_t)j * NB + (size_t)threadIdx.x * PER;
        uint32_t c[PER], sum = 0u;
#pragma unroll
        for (int b = 0; b < PER; b++) { c[b] = h[b]; sum += c[b]; }
        // exclusive scan of the per-thread sums over the CTA
        uint32_t inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += y;
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t excl = inc - sum, total = 0u;
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) {
            if (w < warp) excl += s_warp[w];
            total += s_warp[w];
        }
        if (PASS == 1) {
            if (threadIdx.x == 0) {
                s_n = total;
                if (total > 0u) {
                    float gamma;
                    cz_index(total, 2.f, s_rank[0], s_rank[1], gamma);
                    cz_index(total, 98.f, s_rank[2], s_rank[3], gamma);
                }
            }
            __syncthreads();
            if (s_n == 0u) break;
        }
#pragma unroll
        for (int t = 0; t < kTargets; t++) {
            const uint32_t r = s_rank[t];
            if (s_slot[t] == (uint32_t)j && r >= excl && r - excl < sum) {
                uint32_t acc = excl;
#pragma unroll
                for (int b = 0; b < PER; b++) {
                    if (r >= acc && r - acc < c[b]) { s_bin[t] = threadIdx.x * PER + b; s_res[t] = r - acc; }
                    acc += c[b];
                }
            }
        }
        __syncthreads();                                   // s_warp is rewritten by the next slot's scan
    }
    if (threadIdx.x != 0) return;
    if (PASS == 1 && s_n == 0u) {                          // no valid pixel: nothing to select, (vmin, vmax) = NaN
        const float nan = __uint_as_float(0x7fc00000u);
        S.n = 0u; S.nslots = 0u; S.vmin = nan; S.vmax = nan;
#pragma unroll
        for (int t = 0; t < kTargets; t++) { S.prefix[t] = kNoPrefix; S.slot[t] = 0u; S.rank[t] = 0u; }
        if (vminmax) { vminmax[2 * f] = nan; vminmax[2 * f + 1] = nan; }
        return;
    }
    uint32_t full[kTargets];
#pragma unroll
    for (int t = 0; t < kTargets; t++)
        full[t] = PASS == 1 ? s_bin[t] : (S.prefix[s_slot[t]] << (PASS == 2 ? 11 : 10)) | s_bin[t];
    if (PASS == 1) S.n = s_n;
    if (PASS < 3) {
        uint32_t pref[kTargets] = {kNoPrefix, kNoPrefix, kNoPrefix, kNoPrefix}, nslots = 0u;
#pragma unroll
        for (int t = 0; t < kTargets; t++) {
            uint32_t j = 0u;
            while (j < nslots && pref[j] != full[t]) j++;
            if (j == nslots) pref[nslots++] = full[t];
            S.slot[t] = j;
            S.rank[t] = s_res[t];
        }
        S.nslots = nslots;
#pragma unroll
        for (int t = 0; t < kTargets; t++) S.prefix[t] = pref[t];
    } else {
        uint32_t lo, hi;
        float g2, g98;
        cz_index(S.n, 2.f, lo, hi, g2);
        cz_index(S.n, 98.f, lo, hi, g98);
        const float vmin = cz_lerp(cz_unkey(full[0]), cz_unkey(full[1]), g2);
        const float vmax = cz_lerp(cz_unkey(full[2]), cz_unkey(full[3]), g98);
        S.vmin = vmin; S.vmax = vmax;
        if (vminmax) { vminmax[2 * f] = vmin; vminmax[2 * f + 1] = vmax; }
    }
}

__device__ __forceinline__ uint32_t cz_rgba(float x, float invalid_val, bool norm, float vmin, float den,
                                            const uint32_t* lut, uint32_t bg) {
    if (x == invalid_val) return bg;
    int i = 0;                                             // vmin == vmax: value * 0 -> first colour; NaN -> first colour
    if (norm) {
        const float t = __fdiv_rn(__fsub_rn(x, vmin), den);
        if (t > 1.f) i = 255;                              // before the scale: t * 256 may overflow
        else if (t >= 0.f) i = min(__float2int_rz(__fmul_rn(t, 256.f)), 255);   // exactly 1.0 -> last colour
    }
    return lut[i];
}

__global__ void __launch_bounds__(kThreads)
k_cz_color(const float* __restrict__ value, const long long HW, const int F, const float invalid_val,
           const uint32_t* __restrict__ lut, const uint32_t bg, const CzState* __restrict__ st, uint32_t* __restrict__ rgba) {
    __shared__ uint32_t s_lut[256];
    s_lut[threadIdx.x] = lut[threadIdx.x];
    __syncthreads();
    for (int f = blockIdx.y; f < F; f += gridDim.y) {
        const float vmin = st[f].vmin, vmax = st[f].vmax;
        const bool norm = vmin != vmax;
        const float den = __fsub_rn(vmax, vmin);
        const float* v = value + (size_t)f * (size_t)HW;
        uint32_t* o = rgba + (size_t)f * (size_t)HW;
        const long long stride = (long long)gridDim.x * kThreads;
        if (((reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(o)) & 15) == 0) {
            const long long quads = HW >> 2;             // 128-bit load and store per 4 pixels, then the 0-3 left over
            for (long long g = (long long)blockIdx.x * kThreads + threadIdx.x; g < quads; g += stride) {
                const float4 x = __ldg(reinterpret_cast<const float4*>(v) + g);
                reinterpret_cast<uint4*>(o)[g] = make_uint4(cz_rgba(x.x, invalid_val, norm, vmin, den, s_lut, bg),
                                                            cz_rgba(x.y, invalid_val, norm, vmin, den, s_lut, bg),
                                                            cz_rgba(x.z, invalid_val, norm, vmin, den, s_lut, bg),
                                                            cz_rgba(x.w, invalid_val, norm, vmin, den, s_lut, bg));
            }
            if (blockIdx.x == 0 && threadIdx.x < (HW & 3)) {
                const long long p = quads * 4 + threadIdx.x;
                o[p] = cz_rgba(v[p], invalid_val, norm, vmin, den, s_lut, bg);
            }
        } else {
            for (long long p = (long long)blockIdx.x * kThreads + threadIdx.x; p < HW; p += stride)
                o[p] = cz_rgba(v[p], invalid_val, norm, vmin, den, s_lut, bg);
        }
    }
}

int grid_x(long long groups, int groups_per_thread) {
    const long long per_cta = (long long)kThreads * groups_per_thread;
    return (int)((groups + per_cta - 1) / per_cta);
}

}  // namespace

size_t gs_colorize_scratch_bytes_impl(int F) { return (size_t)F * (kFrameWords * sizeof(uint32_t) + sizeof(CzState)); }

int gs_launch_colorize(int F, int H, int W, const float* value, float invalid_val, const uint32_t* lut, uint32_t bg,
                       void* scratch, uint32_t* rgba, float* vminmax, cudaStream_t s) {
    const long long HW = (long long)H * W;
    const long long groups = (HW + 3) >> 2;
    uint32_t* bins = static_cast<uint32_t*>(scratch);
    CzState* st = reinterpret_cast<CzState*>(bins + (size_t)F * kFrameWords);
    cudaError_t e = cudaMemsetAsync(bins, 0, (size_t)F * kFrameWords * sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    const dim3 gh(grid_x(groups, kGroupsPerThreadHist), F < 65535 ? F : 65535);
    const dim3 gc(grid_x(groups, kGroupsPerThreadColor), F < 65535 ? F : 65535);
    k_cz_hist<1><<<gh, kThreads, 0, s>>>(value, HW, F, invalid_val, bins, st);
    k_cz_select<1><<<F, kThreads, 0, s>>>(bins, st, vminmax);
    k_cz_hist<2><<<gh, kThreads, 0, s>>>(value, HW, F, invalid_val, bins, st);
    k_cz_select<2><<<F, kThreads, 0, s>>>(bins, st, vminmax);
    k_cz_hist<3><<<gh, kThreads, 0, s>>>(value, HW, F, invalid_val, bins, st);
    k_cz_select<3><<<F, kThreads, 0, s>>>(bins, st, vminmax);
    k_cz_color<<<gc, kThreads, 0, s>>>(value, HW, F, invalid_val, lut, bg, st, rgba);
    return 0;
}
