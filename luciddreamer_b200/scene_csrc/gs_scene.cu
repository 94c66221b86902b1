// Training-scene images on the device (include/gsscene.h): the composited camera image and its Canny mask for every
// frame of a scene. One pixel per thread; the frames of a call share one index space p = (f * H + y) * W + x, and
// every neighbourhood stays inside its frame.
//
// Launch sequence (no host loop, so the call is capturable):
//   k_composite  frame bytes -> original_image, and the bytes Canny reads (packed r | g << 8 | b << 16)
//   k_gradient   3x3 Sobel per channel, replicated borders; the channel with the largest |dx| + |dy|
//   k_classify   non-maximum suppression and the two thresholds: none / candidate / strong
//   k_union      union-find over 8-connected candidates (each pixel links to its W, NW, N and NE neighbours)
//   k_resolve    path compression; strong pixels mark their component's root
//   k_output     canny_mask = 0 on a candidate whose root is marked, else 1
// The union-find links by atomicMin, so every component ends at its smallest pixel index whatever the scheduling.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gsscene.h"

namespace {

constexpr int BLOCK = 256;
constexpr int LOW = 50, HIGH = 150;          // image2canny's cv2.Canny(u8, 50, 150)
constexpr int TG22 = 13573;                  // OpenCV's round(tan(22.5 deg) * 2^15)
enum : uint8_t { NONE = 0, CANDIDATE = 1, STRONG = 2 };

struct Dims {
    int H, W;
    int n;                                   // F * H * W
};

__device__ __forceinline__ int px_x(const Dims& d, int p) { return p % d.W; }
__device__ __forceinline__ int px_y(const Dims& d, int p) { return (p / d.W) % d.H; }

__global__ void k_composite(const uint8_t* __restrict__ frames, int C, double bg, Dims d, float* __restrict__ image,
                            uint32_t* __restrict__ rgb) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.n) return;
    const uint8_t* u = frames + (int64_t)p * C;
    const double a = (C == 4 ? u[3] : 255) / 255.0;
    const double ia = 1.0 - a;
    const int64_t hw = (int64_t)d.H * d.W, f = p / hw, at = p - f * hw;
    uint32_t packed = 0;
    for (int c = 0; c < 3; ++c) {
        const double v = u[c] / 255.0 * a + bg * ia;                 // --fmad=false: two products, then the sum
        const float x = fminf(fmaxf((float)v, 0.0f), 1.0f);
        image[(f * 3 + c) * hw + at] = x;
        packed |= (uint32_t)(uint8_t)(x * 255.0f) << (8 * c);        // numpy's astype(np.uint8) truncates
    }
    rgb[p] = packed;
}

__global__ void k_gradient(const uint32_t* __restrict__ rgb, Dims d, int* __restrict__ mag, int* __restrict__ grad) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.n) return;
    const int x = px_x(d, p), y = px_y(d, p), row0 = p - x - y * d.W;
    const int xs[3] = {x > 0 ? x - 1 : 0, x, x < d.W - 1 ? x + 1 : d.W - 1};
    const int ys[3] = {y > 0 ? y - 1 : 0, y, y < d.H - 1 ? y + 1 : d.H - 1};
    uint32_t v[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) v[i][j] = rgb[row0 + ys[i] * d.W + xs[j]];
    int best = -1, bdx = 0, bdy = 0;
    for (int c = 0; c < 3; ++c) {
        auto at = [&](int i, int j) { return (int)((v[i][j] >> (8 * c)) & 255u); };
        const int dx = (at(0, 2) + 2 * at(1, 2) + at(2, 2)) - (at(0, 0) + 2 * at(1, 0) + at(2, 0));
        const int dy = (at(2, 0) + 2 * at(2, 1) + at(2, 2)) - (at(0, 0) + 2 * at(0, 1) + at(0, 2));
        const int m = abs(dx) + abs(dy);
        if (m > best) { best = m; bdx = dx; bdy = dy; }           // strict: ties keep the lowest channel
    }
    mag[p] = best;
    grad[p] = (int)(((uint32_t)bdx & 0xffffu) | ((uint32_t)bdy << 16));   // dx in the low half, dy in the high
}

__device__ __forceinline__ int mag_at(const int* mag, const Dims& d, int p, int x, int y, int dx, int dy) {
    const int xx = x + dx, yy = y + dy;
    if (xx < 0 || xx >= d.W || yy < 0 || yy >= d.H) return 0;
    return mag[p + dy * d.W + dx];
}

__global__ void k_classify(const int* __restrict__ mag, const int* __restrict__ grad, Dims d,
                           uint8_t* __restrict__ kind, int* __restrict__ lab, int* __restrict__ hit) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.n) return;
    const int x = px_x(d, p), y = px_y(d, p), m = mag[p];
    uint8_t k = NONE;
    if (m > LOW) {
        const int g = grad[p];
        const int gx = (int16_t)(g & 0xffff), gy = g >> 16;
        const int ax = abs(gx), ay = abs(gy) << 15;
        const int tg22x = ax * TG22;
        bool peak;
        if (ay < tg22x) {                                              // horizontal gradient: left / right
            peak = m > mag_at(mag, d, p, x, y, -1, 0) && m >= mag_at(mag, d, p, x, y, 1, 0);
        } else if (ay > tg22x + (ax << 16)) {                          // vertical gradient: up / down
            peak = m > mag_at(mag, d, p, x, y, 0, -1) && m >= mag_at(mag, d, p, x, y, 0, 1);
        } else {                                                       // diagonal: the sign of dx * dy picks it
            const int s = (gx ^ gy) < 0 ? -1 : 1;
            peak = m > mag_at(mag, d, p, x, y, -s, -1) && m > mag_at(mag, d, p, x, y, s, 1);
        }
        if (peak) k = m > HIGH ? STRONG : CANDIDATE;
    }
    kind[p] = k;
    lab[p] = p;
    hit[p] = 0;
}

__device__ __forceinline__ int find_root(const int* lab, int x) {
    int y = __ldcg(lab + x);                                           // L2: other SMs' atomicMin land there
    while (y != x) { x = y; y = __ldcg(lab + x); }
    return x;
}

__device__ void unite(int* lab, int a, int b) {
    for (;;) {
        a = find_root(lab, a);
        b = find_root(lab, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(lab + b, a);                         // link the larger root under the smaller
        if (old == b) return;
        b = old;                                                       // b was linked meanwhile: retry from there
    }
}

__global__ void k_union(const uint8_t* __restrict__ kind, Dims d, int* lab) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.n || kind[p] == NONE) return;
    const int x = px_x(d, p), y = px_y(d, p);
    if (x > 0 && kind[p - 1] != NONE) unite(lab, p, p - 1);
    if (y > 0) {
        const int q = p - d.W;
        if (x > 0 && kind[q - 1] != NONE) unite(lab, p, q - 1);
        if (kind[q] != NONE) unite(lab, p, q);
        if (x < d.W - 1 && kind[q + 1] != NONE) unite(lab, p, q + 1);
    }
}

__global__ void k_resolve(const uint8_t* __restrict__ kind, Dims d, int* lab, int* hit) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.n || kind[p] == NONE) return;
    const int r = find_root(lab, p);
    lab[p] = r;
    if (kind[p] == STRONG) atomicOr(hit + r, 1);
}

__global__ void k_output(const uint8_t* __restrict__ kind, const int* __restrict__ lab, const int* __restrict__ hit,
                         Dims d, float* __restrict__ canny) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.n) return;
    canny[p] = (kind[p] != NONE && hit[lab[p]]) ? 0.0f : 1.0f;
}

// ---- scratch layout: rgb is dead once k_gradient has run, so the component marks reuse it
struct Layout {
    size_t rgb, mag, grad, lab, kind, total;
};

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

Layout layout(int64_t n) {
    Layout L{};
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes); return at; };
    const int64_t nn = n > 0 ? n : 1;
    L.rgb = take(4 * nn); L.mag = take(4 * nn); L.grad = take(4 * nn); L.lab = take(4 * nn); L.kind = take(nn);
    L.total = o;
    return L;
}

bool sizes_ok(int F, int H, int W) {
    return F >= 0 && H >= 1 && W >= 1 && (int64_t)F * H * W <= (int64_t)INT32_MAX - BLOCK;
}

bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

}  // namespace

extern "C" {

int gsscene_abi_version(void) { return 1; }

int gsscene_scratch_bytes(int32_t F, int32_t H, int32_t W, uint64_t* bytes) {
    if (!bytes || !sizes_ok(F, H, W)) return GSSCENE_EINVAL;
    *bytes = layout((int64_t)F * H * W).total;
    return GSSCENE_OK;
}

int gsscene_camera_images(const uint8_t* frames, int32_t F, int32_t H, int32_t W, int32_t C, int32_t white_background,
                          float* image, float* canny_mask, void* scratch, uint64_t scratch_bytes, void* stream) {
    if (!sizes_ok(F, H, W) || (C != 3 && C != 4) || (white_background != 0 && white_background != 1))
        return GSSCENE_EINVAL;
    if (!frames || !image || !aligned(image, 4) || !canny_mask || !aligned(canny_mask, 4)) return GSSCENE_EINVAL;
    const int64_t n = (int64_t)F * H * W;
    const Layout L = layout(n);
    if (!scratch || !aligned(scratch, 256) || scratch_bytes < L.total) return GSSCENE_EINVAL;
    if (n == 0) return GSSCENE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    char* s = (char*)scratch;
    uint32_t* rgb = (uint32_t*)(s + L.rgb);
    int* mag = (int*)(s + L.mag);
    int* grad = (int*)(s + L.grad);
    int* lab = (int*)(s + L.lab);
    int* hit = (int*)(s + L.rgb);
    uint8_t* kind = (uint8_t*)(s + L.kind);
    const Dims d{H, W, (int)n};
    const int grid = (int)((n + BLOCK - 1) / BLOCK);
    k_composite<<<grid, BLOCK, 0, st>>>(frames, C, white_background ? 1.0 : 0.0, d, image, rgb);
    k_gradient<<<grid, BLOCK, 0, st>>>(rgb, d, mag, grad);
    k_classify<<<grid, BLOCK, 0, st>>>(mag, grad, d, kind, lab, hit);
    k_union<<<grid, BLOCK, 0, st>>>(kind, d, lab);
    k_resolve<<<grid, BLOCK, 0, st>>>(kind, d, lab, hit);
    k_output<<<grid, BLOCK, 0, st>>>(kind, lab, hit, d, canny_mask);
    return cudaPeekAtLastError() == cudaSuccess ? GSSCENE_OK : GSSCENE_ECUDA;
}

}  // extern "C"
