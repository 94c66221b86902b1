// Densification and pruning of a Gaussian model on the device (include/gsdensify.h), restating the reference
// GaussianModel's densify_and_prune (densify_and_clone, densify_and_split, prune_points) and reset_opacity op for op.
//
// Launch sequence of a densify:
//   k_plan   one row per thread: the clone / split / prune decisions as flags, and per block the number of rows each
//            output segment receives (five counters packed 12 bits apiece into one 64-bit word)
//   k_scan   one CTA: exclusive offsets of every block in every segment, the totals and counts[4]
//   k_map    one row per thread: the block's exclusive scan of the flags, the output rows the row fills, and the
//            split rows' stds
//   k_apply  one float per thread over every output tensor: the gather, the split rows' xyz and scaling, zero moments
// Built with --fmad=false: torch evaluates every product and sum of these expressions as its own element-wise op, so
// each one is rounded on its own here too. The only fused multiply-adds are the ones written out (the bmm of the
// split rows' xyz) and those inside expf, logf and the IEEE division.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/gsdensify.h"

namespace {

constexpr int BLOCK = 256;
constexpr int SCAN_THREADS = 1024;
constexpr int APPLY_PER_BLOCK = 4 * BLOCK;          // floats of one tensor per k_apply block

// densify_and_split(N=2): the split copies' scaling is divided by 0.8 * N, which ATen's true-divide by a CPU scalar
// evaluates as a product with the float reciprocal of float32(1.6)
constexpr float SPLIT_INV = 1.0f / 1.6f;
// reset_opacity: torch.ones_like(x) * 0.01
constexpr float RESET_CAP = 0.01f;

enum : uint8_t { CLONE = 1, SPLIT = 2, KEEP = 4, KEEP_SPLIT = 8 };

// the five per-row counters: surviving originals, kept clones, kept split pairs, splits (kept or not), clones
enum { F_ORIG = 0, F_CLONE = 1, F_SPLIT_KEPT = 2, F_SPLIT = 3, F_CLONES = 4, NF = 5 };
constexpr int FIELD_BITS = 12;                      // a block holds at most 256 rows

__device__ __forceinline__ uint64_t pack(uint8_t f) {
    const uint64_t orig = !(f & SPLIT) && (f & KEEP), clone = (f & CLONE) && (f & KEEP);
    const uint64_t split_kept = (f & SPLIT) && (f & KEEP_SPLIT), split = (f & SPLIT) != 0, clones = (f & CLONE) != 0;
    return orig | clone << FIELD_BITS | split_kept << (2 * FIELD_BITS) | split << (3 * FIELD_BITS) |
           clones << (4 * FIELD_BITS);
}

__device__ __forceinline__ int field(uint64_t v, int k) { return (int)((v >> (k * FIELD_BITS)) & 0xfff); }

// torch.max over a dim and torch.minimum propagate NaN
__device__ __forceinline__ float tmax(float a, float b) { return (isnan(a) || a > b) ? a : b; }
__device__ __forceinline__ float tmin(float a, float b) { return (isnan(a) || a < b) ? a : b; }

// torch.sigmoid: 1 / (1 + exp(-x))
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// exclusive scan of one 64-bit word per thread over a BLOCK-thread CTA; *total gets the CTA's sum
__device__ uint64_t block_exclusive_scan(uint64_t v, uint64_t* total) {
    __shared__ uint64_t warp_sum[BLOCK / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = lane < BLOCK / 32 ? warp_sum[lane] : 0;
#pragma unroll
        for (int o = 1; o < BLOCK / 32; o <<= 1) {
            const uint64_t y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < BLOCK / 32) warp_sum[lane] = w;
    }
    __syncthreads();
    *total = warp_sum[BLOCK / 32 - 1];
    return (warp ? warp_sum[warp - 1] : 0) + x - v;
}

struct Plan {
    float max_grad, dense_scale, min_opacity, max_screen, world_scale;
    int screen;
};

__global__ void k_plan(int P, const float* __restrict__ accum, const float* __restrict__ denom,
                       const float* __restrict__ scaling, const float* __restrict__ opacity, Plan pl,
                       uint8_t* __restrict__ flags, uint64_t* __restrict__ block_sum) {
    const int i = blockIdx.x * BLOCK + threadIdx.x;
    uint8_t f = 0;
    if (i < P) {
        float g = accum[i] / denom[i];                              // grads = accum / denom; grads[isnan] = 0
        if (isnan(g)) g = 0.f;
        const float s0 = expf(scaling[3 * i]), s1 = expf(scaling[3 * i + 1]), s2 = expf(scaling[3 * i + 2]);
        const float smax = tmax(tmax(s0, s1), s2);
        // densify_and_clone: torch.norm over the size-1 dim is |g| on the device, also where g * g would
        // underflow or overflow (DESIGN section 7)
        if (fabsf(g) >= pl.max_grad && smax <= pl.dense_scale) f |= CLONE;
        // densify_and_split: the padded gradient is g for every original row and 0 for the clones, whose scaling
        // is their source's and so never above dense_scale
        if (g >= pl.max_grad && smax > pl.dense_scale) f |= SPLIT;
        // the final prune, on the originals and clones as they are and on the split copies' new scaling
        const bool transparent = sigmoid(opacity[i]) < pl.min_opacity;
        const bool screen_all = pl.screen && 0.f > pl.max_screen;    // max_radii2D is all zero by then
        if (!(transparent || screen_all || (pl.screen && smax > pl.world_scale))) f |= KEEP;
        const float n0 = expf(logf(s0 * SPLIT_INV)), n1 = expf(logf(s1 * SPLIT_INV)), n2 = expf(logf(s2 * SPLIT_INV));
        if (!(transparent || screen_all || (pl.screen && tmax(tmax(n0, n1), n2) > pl.world_scale))) f |= KEEP_SPLIT;
        flags[i] = f;
    }
    uint64_t total;
    block_exclusive_scan(pack(f), &total);
    if (threadIdx.x == 0) block_sum[blockIdx.x] = total;
}

// one CTA: block_off[b] = exclusive offsets of block b in the first four fields; totals[NF]; counts[4]
__global__ void __launch_bounds__(SCAN_THREADS) k_scan(int nb, const uint64_t* __restrict__ block_sum,
                                                       int4* __restrict__ block_off, int* __restrict__ totals,
                                                       int* __restrict__ counts) {
    __shared__ int warp_sum[NF][SCAN_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int chunk = (nb + SCAN_THREADS - 1) / SCAN_THREADS;
    const int b0 = min(nb, t * chunk), b1 = min(nb, b0 + chunk);
    int own[NF] = {0, 0, 0, 0, 0};
    for (int b = b0; b < b1; b++)
        for (int k = 0; k < NF; k++) own[k] += field(block_sum[b], k);
    int excl[NF];
    for (int k = 0; k < NF; k++) {
        int x = own[k];
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sum[k][warp] = x;
        excl[k] = x - own[k];
    }
    __syncthreads();
    if (warp == 0) {
        for (int k = 0; k < NF; k++) {
            int w = warp_sum[k][lane];
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            warp_sum[k][lane] = w;
        }
    }
    __syncthreads();
    for (int k = 0; k < NF; k++) excl[k] += warp ? warp_sum[k][warp - 1] : 0;
    for (int b = b0; b < b1; b++) {
        block_off[b] = make_int4(excl[0], excl[1], excl[2], excl[3]);
        for (int k = 0; k < NF; k++) excl[k] += field(block_sum[b], k);
    }
    if (t == 0) {
        int tot[NF];
        for (int k = 0; k < NF; k++) tot[k] = warp_sum[k][SCAN_THREADS / 32 - 1];
        for (int k = 0; k < NF; k++) totals[k] = tot[k];
        counts[0] = tot[F_CLONES];
        counts[1] = tot[F_SPLIT];
        counts[2] = tot[F_ORIG];
        counts[3] = tot[F_ORIG] + tot[F_CLONE] + 2 * tot[F_SPLIT_KEPT];
    }
}

// map[o] = {source row, kind}: kind -2 original, -1 clone, k >= 0 the split copy drawing sample row k
__global__ void k_map(int P, const uint8_t* __restrict__ flags, const int4* __restrict__ block_off,
                      const int* __restrict__ totals, const float* __restrict__ scaling, int S, int2* __restrict__ map,
                      float* __restrict__ stds) {
    const int i = blockIdx.x * BLOCK + threadIdx.x;
    const uint8_t f = i < P ? flags[i] : 0;
    uint64_t total;
    const uint64_t ex = block_exclusive_scan(pack(f), &total);
    if (i >= P) return;
    const int4 bo = block_off[blockIdx.x];
    const int n_orig = totals[F_ORIG], n_clone = totals[F_CLONE], n_split = totals[F_SPLIT_KEPT];
    if (!(f & SPLIT) && (f & KEEP)) map[bo.x + field(ex, F_ORIG)] = make_int2(i, -2);
    if ((f & CLONE) && (f & KEEP)) map[n_orig + bo.y + field(ex, F_CLONE)] = make_int2(i, -1);
    if (f & SPLIT) {
        const int k = bo.w + field(ex, F_SPLIT);                   // the row's rank among the selected ones
        for (int c = 0; c < 3; c++) stds[3 * k + c] = stds[3 * (S + k) + c] = expf(scaling[3 * i + c]);
        if (f & KEEP_SPLIT) {
            const int o = n_orig + n_clone + bo.z + field(ex, F_SPLIT_KEPT);
            map[o] = make_int2(i, k);
            map[o + n_split] = make_int2(i, S + k);
        }
    }
}

struct Tensors {
    const float* src[GSDENSIFY_MAX_TENSORS];
    float* dst[GSDENSIFY_MAX_TENSORS];
    int width[GSDENSIFY_MAX_TENSORS];
    int kind[GSDENSIFY_MAX_TENSORS];
    int first_block[GSDENSIFY_MAX_TENSORS + 1];
    int n;
};

// torch.bmm over the 2S split rows: cuBLAS runs the batch in chunks of 65 535 matrices, and on the H100 the kernel it
// picks for a chunk of 12 998 to 37 292 matrices adds the last two products of each 3x3 @ 3x1 product in the other
// order than the kernel it picks for every other chunk size (probed for every chunk size up to 65 535, DESIGN
// section 7)
constexpr int BMM_CHUNK = 65535;
constexpr int BMM_SWAP_LO = 12998, BMM_SWAP_HI = 37292;

__device__ __forceinline__ bool bmm_swapped(int k, int batch) {
    const int c = min(BMM_CHUNK, batch - k / BMM_CHUNK * BMM_CHUNK);          // size of the chunk holding matrix k
    return c >= BMM_SWAP_LO && c <= BMM_SWAP_HI;
}

// row c of utils.general.build_rotation(r) @ s, as torch evaluates it: the quaternion normalised by the square root
// of the left-to-right sum of squares, each entry its own chain of element-wise ops, and the row's dot product as
// cuBLAS rounds it: fma(m1, s1, m0 * s0) + m2 * s2, or fma(m2, s2, m0 * s0) + m1 * s1 when `swapped`
__device__ float rotate_row(const float* __restrict__ q4, const float* __restrict__ s, int c, bool swapped) {
    const float a = q4[0], b = q4[1], d = q4[2], e = q4[3];
    const float norm = sqrtf(a * a + b * b + d * d + e * e);
    const float r = a / norm, x = b / norm, y = d / norm, z = e / norm;
    float m0, m1, m2;
    if (c == 0) {
        m0 = 1.f - 2.f * (y * y + z * z);
        m1 = 2.f * (x * y - r * z);
        m2 = 2.f * (x * z + r * y);
    } else if (c == 1) {
        m0 = 2.f * (x * y + r * z);
        m1 = 1.f - 2.f * (x * x + z * z);
        m2 = 2.f * (y * z - r * x);
    } else {
        m0 = 2.f * (x * z - r * y);
        m1 = 2.f * (y * z + r * x);
        m2 = 1.f - 2.f * (x * x + y * y);
    }
    return swapped ? __fmaf_rn(m2, s[2], m0 * s[0]) + m1 * s[1] : __fmaf_rn(m1, s[1], m0 * s[0]) + m2 * s[2];
}

__global__ void k_apply(const int2* __restrict__ map, Tensors T, const float* __restrict__ rotation,
                        const float* __restrict__ samples, int batch, unsigned total_rows) {
    int t = 0;
    while (t + 1 < T.n && (int)blockIdx.x >= T.first_block[t + 1]) t++;
    const unsigned w = (unsigned)T.width[t], n = total_rows * w;
    const unsigned base = (unsigned)(blockIdx.x - T.first_block[t]) * APPLY_PER_BLOCK;
    const float* __restrict__ src = T.src[t];
    float* __restrict__ dst = T.dst[t];
    const int kind = T.kind[t];
#pragma unroll
    for (int j = 0; j < APPLY_PER_BLOCK / BLOCK; j++) {
        const unsigned e = base + j * BLOCK + threadIdx.x;
        if (e >= n) break;
        const unsigned o = e / w, c = e - o * w;
        const int2 m = map[o];
        const float v = src[(size_t)m.x * w + c];
        float out = v;
        if (kind == GSDENSIFY_MOMENT) {
            out = m.y == -2 ? v : 0.f;
        } else if (m.y >= 0) {
            if (kind == GSDENSIFY_XYZ)
                out = rotate_row(rotation + 4 * (size_t)m.x, samples + 3 * (size_t)m.y, (int)c,
                                 bmm_swapped(m.y, batch)) + v;
            else if (kind == GSDENSIFY_SCALING)
                out = logf(expf(v) * SPLIT_INV);
        }
        dst[e] = out;
    }
}

// reset_opacity: inverse_sigmoid(min(sigmoid(o), 0.01)) = log(x / (1 - x)); the moments start again from zero
__global__ void k_reset_opacity(int P, const float* __restrict__ opacity, float* __restrict__ out,
                                float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq) {
    const int i = blockIdx.x * BLOCK + threadIdx.x;
    if (i >= P) return;
    const float x = tmin(sigmoid(opacity[i]), RESET_CAP);
    out[i] = logf(x / (1.f - x));
    if (exp_avg) exp_avg[i] = 0.f;
    if (exp_avg_sq) exp_avg_sq[i] = 0.f;
}

struct Layout {
    size_t flags, block_sum, block_off, totals, total;
};

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

int blocks(int P) { return (P + BLOCK - 1) / BLOCK; }

Layout layout(int P) {
    Layout L{};
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes); return at; };
    const size_t nb = (size_t)(blocks(P) > 0 ? blocks(P) : 1);
    L.flags = take(P > 0 ? P : 1);
    L.block_sum = take(8 * nb);
    L.block_off = take(16 * nb);
    L.totals = take(4 * 8);
    L.total = o;
    return L;
}

bool size_ok(int P) { return P >= 0 && P < (1 << 30); }

bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

bool scratch_ok(int P, const void* scratch, uint64_t bytes) {
    return scratch && aligned(scratch, 256) && bytes >= layout(P).total;
}

int launched() { return cudaPeekAtLastError() == cudaSuccess ? GSDENSIFY_OK : GSDENSIFY_ECUDA; }

}  // namespace

extern "C" {

int gsdensify_abi_version(void) { return 1; }

int gsdensify_scratch_bytes(int32_t P, uint64_t* bytes) {
    if (!bytes || !size_ok(P)) return GSDENSIFY_EINVAL;
    *bytes = layout(P).total;
    return GSDENSIFY_OK;
}

int gsdensify_plan(int32_t P, const float* accum, const float* denom, const float* scaling, const float* opacity,
                   float max_grad, float dense_scale, float min_opacity, int32_t screen, float max_screen,
                   float world_scale, int32_t* counts, void* scratch, uint64_t scratch_bytes, void* stream) {
    if (!size_ok(P) || (screen != 0 && screen != 1) || !counts || !aligned(counts, 4)) return GSDENSIFY_EINVAL;
    if (!scratch_ok(P, scratch, scratch_bytes)) return GSDENSIFY_EINVAL;
    if (P > 0 && (!accum || !denom || !scaling || !opacity)) return GSDENSIFY_EINVAL;
    const Layout L = layout(P);
    char* s = (char*)scratch;
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = blocks(P);
    const Plan pl{max_grad, dense_scale, min_opacity, max_screen, world_scale, screen};
    if (nb > 0)
        k_plan<<<nb, BLOCK, 0, st>>>(P, accum, denom, scaling, opacity, pl, (uint8_t*)(s + L.flags),
                                     (uint64_t*)(s + L.block_sum));
    k_scan<<<1, SCAN_THREADS, 0, st>>>(nb, (const uint64_t*)(s + L.block_sum), (int4*)(s + L.block_off),
                                       (int*)(s + L.totals), counts);
    return launched();
}

int gsdensify_map(int32_t P, const float* scaling, int32_t S, int32_t P_new, int32_t* map, float* stds, void* scratch,
                  uint64_t scratch_bytes, void* stream) {
    if (!size_ok(P) || S < 0 || S > P || P_new < 0 || (int64_t)P_new > 2 * (int64_t)P)
        return GSDENSIFY_EINVAL;
    if (!scratch_ok(P, scratch, scratch_bytes)) return GSDENSIFY_EINVAL;
    if ((P > 0 && !scaling) || (P_new > 0 && (!map || !aligned(map, 8))) || (S > 0 && (!stds || !aligned(stds, 4))))
        return GSDENSIFY_EINVAL;
    if (P == 0) return GSDENSIFY_OK;
    const Layout L = layout(P);
    char* s = (char*)scratch;
    k_map<<<blocks(P), BLOCK, 0, (cudaStream_t)stream>>>(P, (const uint8_t*)(s + L.flags),
                                                         (const int4*)(s + L.block_off), (const int*)(s + L.totals),
                                                         scaling, S, (int2*)map, stds);
    return launched();
}

int gsdensify_apply(const int32_t* map, int32_t P_new, const gsdensify_tensor* tensors, int32_t n,
                    const float* rotation, const float* samples, int32_t S, void* stream) {
    if (P_new < 0 || S < 0 || S >= (1 << 30) || n < 0 || n > GSDENSIFY_MAX_TENSORS || (n > 0 && !tensors)) return GSDENSIFY_EINVAL;
    if (P_new > 0 && (!map || !aligned(map, 8))) return GSDENSIFY_EINVAL;
    Tensors T{};
    int64_t nblk = 0;
    bool xyz = false;
    for (int k = 0; k < n; k++) {
        const gsdensify_tensor& t = tensors[k];
        if (t.width < 1 || t.kind < GSDENSIFY_PARAM || t.kind > GSDENSIFY_MOMENT) return GSDENSIFY_EINVAL;
        if ((int64_t)P_new * t.width >= INT32_MAX) return GSDENSIFY_EINVAL;
        if (P_new > 0 && (!t.src || !t.dst || !aligned(t.src, 4) || !aligned(t.dst, 4))) return GSDENSIFY_EINVAL;
        if (t.kind == GSDENSIFY_XYZ && t.width != 3) return GSDENSIFY_EINVAL;
        if (t.kind == GSDENSIFY_SCALING && t.width != 3) return GSDENSIFY_EINVAL;
        xyz |= t.kind == GSDENSIFY_XYZ;
        T.src[k] = t.src;
        T.dst[k] = t.dst;
        T.width[k] = t.width;
        T.kind[k] = t.kind;
        T.first_block[k] = (int)nblk;
        nblk += ((int64_t)P_new * t.width + APPLY_PER_BLOCK - 1) / APPLY_PER_BLOCK;
        if (nblk >= INT32_MAX) return GSDENSIFY_EINVAL;
    }
    if (xyz && P_new > 0 && (!rotation || !aligned(rotation, 4) || (S > 0 && (!samples || !aligned(samples, 4)))))
        return GSDENSIFY_EINVAL;
    T.first_block[n] = (int)nblk;
    T.n = n;
    if (nblk == 0) return GSDENSIFY_OK;
    k_apply<<<(unsigned)nblk, BLOCK, 0, (cudaStream_t)stream>>>((const int2*)map, T, rotation, samples,
                                                                2 * S, (unsigned)P_new);
    return launched();
}

int gsdensify_reset_opacity(int32_t P, const float* opacity, float* out, float* exp_avg, float* exp_avg_sq,
                            void* stream) {
    if (!size_ok(P)) return GSDENSIFY_EINVAL;
    if (P > 0 && (!opacity || !out || !aligned(opacity, 4) || !aligned(out, 4))) return GSDENSIFY_EINVAL;
    if ((exp_avg && !aligned(exp_avg, 4)) || (exp_avg_sq && !aligned(exp_avg_sq, 4))) return GSDENSIFY_EINVAL;
    if (P == 0) return GSDENSIFY_OK;
    k_reset_opacity<<<blocks(P), BLOCK, 0, (cudaStream_t)stream>>>(P, opacity, out, exp_avg, exp_avg_sq);
    return launched();
}

}  // extern "C"
