// Point-cloud warp into camera views (include/gspcd.h): LucidDreamer.generate_pcd's project / griddata-linear /
// edge ring / max-min filter chain on the device. Per view: project and compact the valid points in index order,
// write the round mask, bin the points into a uniform cell grid (counting sort, ascending index within a cell),
// filter the mask, locate the Delaunay triangle of every pixel that needs a value, then assemble the frame with
// the reference's own expressions. The grow stage (gspcd_grow_view) reuses the grid, hull and locate steps on the
// border points of a view. No float atomics; every result is independent of thread scheduling.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gspcd.h"
#include "gs_pcd_geom.cuh"

namespace {

constexpr int SCAN_BLOCK = 1024;

struct Cam { double R[9], T[3], K[9]; };

__device__ __forceinline__ bool project(const double* __restrict__ pts, int64_t n, int64_t i, const Cam& c, int W,
                                        int H, double& u, double& v) {
    const double X = pts[i], Y = pts[n + i], Z = pts[2 * n + i];
    double cam[3], pix[3];
    // R.dot(p) + T and K @ cam as numpy's matmul rounds them: fma(r2, z, fma(r1, y, r0 * x)), then + T
#pragma unroll
    for (int r = 0; r < 3; ++r)
        cam[r] = __dadd_rn(__fma_rn(c.R[3 * r + 2], Z, __fma_rn(c.R[3 * r + 1], Y, __dmul_rn(c.R[3 * r], X))), c.T[r]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
        pix[r] = __fma_rn(c.K[3 * r + 2], cam[2], __fma_rn(c.K[3 * r + 1], cam[1], __dmul_rn(c.K[3 * r], cam[0])));
    u = __ddiv_rn(pix[0], pix[2]);
    v = __ddiv_rn(pix[1], pix[2]);
    return pix[2] > 0.0 && u >= 0.0 && u <= (double)(W - 1) && v >= 0.0 && v <= (double)(H - 1);
}

__global__ void k_flags(const double* __restrict__ pts, int64_t n, Cam c, int W, int H, int* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double u, v;
    flags[i] = project(pts, n, i, c, W, H, u, v) ? 1 : 0;
}

// ---- exclusive scan of int32 (block partials, one-block scan of the partials, add back)
__device__ int block_exclusive_scan(int v, int* total) {
    __shared__ int warp_sums[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < (int)(blockDim.x >> 5) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    const int before = warp == 0 ? 0 : warp_sums[warp - 1];
    *total = warp_sums[(blockDim.x >> 5) - 1];
    __syncthreads();
    return before + x - v;
}

__global__ void __launch_bounds__(SCAN_BLOCK) k_scan_blocks(const int* __restrict__ in, int* __restrict__ out,
                                                            int64_t n, int* __restrict__ sums) {
    const int64_t i = (int64_t)blockIdx.x * SCAN_BLOCK + threadIdx.x;
    const int v = i < n ? in[i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, &total);
    if (i < n) out[i] = ex;
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(SCAN_BLOCK) k_scan_sums(int* __restrict__ sums, int nb, int* __restrict__ grand) {
    int carry = 0;
    for (int base = 0; base < nb; base += SCAN_BLOCK) {
        const int i = base + threadIdx.x;
        const int v = i < nb ? sums[i] : 0;
        int total;
        const int ex = block_exclusive_scan(v, &total);
        if (i < nb) sums[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0 && grand) *grand = carry;
}

__global__ void k_scan_add(int* __restrict__ out, int64_t n, const int* __restrict__ sums) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] += sums[i / SCAN_BLOCK];
}

void exclusive_scan(const int* in, int* out, int64_t n, int* sums, int* grand, cudaStream_t st) {
    const int nb = (int)((n + SCAN_BLOCK - 1) / SCAN_BLOCK);
    k_scan_blocks<<<nb, SCAN_BLOCK, 0, st>>>(in, out, n, sums);
    k_scan_sums<<<1, SCAN_BLOCK, 0, st>>>(sums, nb, grand);
    k_scan_add<<<(int)((n + 255) / 256), 256, 0, st>>>(out, n, sums);
}

// ---- compaction: valid points in ascending index order, round mask
__global__ void k_compact(const double* __restrict__ pts, int64_t n, Cam c, int W, int H,
                          const int* __restrict__ flags, const int* __restrict__ pos,
                          int* __restrict__ vidx, double* __restrict__ cx, double* __restrict__ cy,
                          int* __restrict__ rx, int* __restrict__ ry, uint8_t* __restrict__ round_mask) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    double u, v;
    project(pts, n, i, c, W, H, u, v);
    const int j = pos[i];
    const int iu = (int)rint(u), iv = (int)rint(v);                 // np.round: half to even
    vidx[j] = (int)i;
    cx[j] = u; cy[j] = v;
    rx[j] = iu; ry[j] = iv;
    round_mask[(int64_t)iv * W + iu] = 1;
}

struct GridDims { int gw, gh; double s, inv_s; };

GridDims grid_dims(int64_t n, int H, int W) {
    // about two points per cell when the whole cloud lands in the view
    double s = sqrt((double)H * (double)W * 2.0 / (double)(n > 0 ? n : 1));
    if (s < 0.5) s = 0.5;
    const double big = (double)(W > H ? W : H);
    if (s > big) s = big;
    GridDims g;
    g.s = s; g.inv_s = 1.0 / s;
    g.gw = (int)((double)(W - 1) * g.inv_s) + 1;
    g.gh = (int)((double)(H - 1) * g.inv_s) + 1;
    return g;
}

__global__ void k_cell_count(const double* __restrict__ cx, const double* __restrict__ cy,
                             const int* __restrict__ count, GridDims g, int* __restrict__ cell_count) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *count) return;
    const int c = pcd::cell_coord(cy[j], g.inv_s, g.gh) * g.gw + pcd::cell_coord(cx[j], g.inv_s, g.gw);
    atomicAdd(&cell_count[c], 1);
}

__global__ void k_cell_scatter(const double* __restrict__ cx, const double* __restrict__ cy,
                               const int* __restrict__ count, GridDims g, int* __restrict__ cursor,
                               int* __restrict__ sidx) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *count) return;
    const int c = pcd::cell_coord(cy[j], g.inv_s, g.gh) * g.gw + pcd::cell_coord(cx[j], g.inv_s, g.gw);
    sidx[atomicAdd(&cursor[c], 1)] = j;
}

// The scatter's order within a cell depends on scheduling; a heap sort per cell restores index order.
__global__ void k_cell_sort(const int* __restrict__ cell_start, int ncells, int* __restrict__ sidx) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncells) return;
    int* a = sidx + cell_start[c];
    const int m = cell_start[c + 1] - cell_start[c];
    if (m < 2) return;
    auto sift = [&](int root, int end) {
        while (2 * root + 1 < end) {
            int ch = 2 * root + 1;
            if (ch + 1 < end && a[ch] < a[ch + 1]) ++ch;
            if (a[root] >= a[ch]) return;
            int t = a[root]; a[root] = a[ch]; a[ch] = t;
            root = ch;
        }
    };
    for (int r = m / 2 - 1; r >= 0; --r) sift(r, m);
    for (int end = m - 1; end > 0; --end) {
        int t = a[0]; a[0] = a[end]; a[end] = t;
        sift(0, end);
    }
}

__global__ void k_cell_gather(const int* __restrict__ count, const int* __restrict__ sidx,
                              const double* __restrict__ cx, const double* __restrict__ cy,
                              double* __restrict__ sx, double* __restrict__ sy) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= *count) return;
    const int j = sidx[e];
    sx[e] = cx[j]; sy[e] = cy[j];
}

// ---- separable max / min filters, scipy.ndimage mode='reflect' (d c b a | a b c d), any image size
__device__ __forceinline__ int reflect(int i, int n) {
    const int p = 2 * n;
    i %= p;
    if (i < 0) i += p;
    return i < n ? i : p - 1 - i;
}

template <bool MAX, int RADIUS, bool ROWS>
__global__ void k_filter(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int W, int H) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    const int x = (int)(p % W), y = (int)(p / W);
    uint8_t r = MAX ? 0 : 1;
    for (int d = -RADIUS; d <= RADIUS; ++d) {
        const uint8_t v = ROWS ? in[(int64_t)y * W + reflect(x + d, W)] : in[(int64_t)reflect(y + d, H) * W + x];
        r = MAX ? (v > r ? v : r) : (v < r ? v : r);
    }
    out[p] = r;
}

// ---- convex hull: occupied-row/column extents per grid column/row, the candidate cells near them (column-major,
// so that per-column sorts give xy order), then one monotone chain
__global__ void k_extents(const int* __restrict__ cell_start, int gw, int gh, int* __restrict__ top,
                          int* __restrict__ bot, int* __restrict__ left, int* __restrict__ right) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= gw * gh || cell_start[c + 1] == cell_start[c]) return;
    const int i = c % gw, j = c / gw;
    atomicMax(&top[i], j); atomicMin(&bot[i], j); atomicMin(&left[j], i); atomicMax(&right[j], i);
}

__global__ void k_cand_count(const int* __restrict__ cell_start, int gw, int gh, const int* __restrict__ top,
                             const int* __restrict__ bot, const int* __restrict__ left, const int* __restrict__ right,
                             int* __restrict__ cand_count) {
    const int cc = blockIdx.x * blockDim.x + threadIdx.x;        // column-major cell index i * gh + j
    if (cc >= gw * gh) return;
    const int i = cc / gh, j = cc % gh, c = j * gw + i;
    const int m = cell_start[c + 1] - cell_start[c];
    cand_count[cc] = m > 0 && pcd::in_hull_band(i, j, top[i], bot[i], left[j], right[j]) ? m : 0;
}

__global__ void k_cand_gather(const int* __restrict__ cell_start, int gw, int gh, const int* __restrict__ cand_start,
                              int* __restrict__ cand) {
    const int cc = blockIdx.x * blockDim.x + threadIdx.x;
    if (cc >= gw * gh) return;
    const int i = cc / gh, j = cc % gh, c = j * gw + i;
    const int at = cand_start[cc], m = cand_start[cc + 1] - at;
    for (int t = 0; t < m; ++t) cand[at + t] = cell_start[c] + t;
}

// Cell columns partition x monotonically, so sorting each column's candidates sorts them all.
__global__ void k_cand_sort(const int* __restrict__ cand_start, int gw, int gh, const double* __restrict__ x,
                            const double* __restrict__ y, const int* __restrict__ idx, int* __restrict__ cand) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= gw) return;
    int* a = cand + cand_start[i * gh];
    const int m = cand_start[(i + 1) * gh] - cand_start[i * gh];
    auto less = [&](int u, int v) { return pcd::xy_less(pcd::Pt{x[u], y[u]}, idx[u], pcd::Pt{x[v], y[v]}, idx[v]); };
    auto sift = [&](int root, int end) {
        while (2 * root + 1 < end) {
            int ch = 2 * root + 1;
            if (ch + 1 < end && less(a[ch], a[ch + 1])) ++ch;
            if (!less(a[root], a[ch])) return;
            int t = a[root]; a[root] = a[ch]; a[ch] = t;
            root = ch;
        }
    };
    for (int r = m / 2 - 1; r >= 0; --r) sift(r, m);
    for (int end = m - 1; end > 0; --end) {
        int t = a[0]; a[0] = a[end]; a[end] = t;
        sift(0, end);
    }
}

__global__ void k_chain(const double* __restrict__ x, const double* __restrict__ y, const int* __restrict__ cand,
                        const int* __restrict__ n_cand, int* __restrict__ hull, int* __restrict__ hull_n,
                        int* __restrict__ status) {
    int st = 0;
    *hull_n = pcd::monotone_chain(x, y, cand, *n_cand, hull, st);
    if (st) atomicOr(status, st);
}

__device__ __forceinline__ bool ring0(int x, int y, int W, int H) { return x == 0 || y == 0 || x == W - 1 || y == H - 1; }

// The Delaunay triangle of q and its barycentric weights: v[] are the input indices of its vertices. False when q lies
// outside the closed hull (pixels outside it take the fill value without a search), or there are fewer than three
// points, or all are collinear. griddata's linear value is then 0 + l0 * f(v0) + l1 * f(v1) + l2 * f(v2).
__device__ __forceinline__ bool locate_linear(const pcd::Grid& g, int count, const int* hull, int hull_n, pcd::Pt q,
                                              int v[3], double l[3], int& st) {
    pcd::Located t{{-1, -1, -1}};
    if (pcd::in_hull(g.x, g.y, hull, hull_n, q, st)) t = pcd::locate(g, count, q, st);
    if (t.v[0] < 0) return false;
    const pcd::Pt a = {g.x[t.v[0]], g.y[t.v[0]]}, b = {g.x[t.v[1]], g.y[t.v[1]]}, c = {g.x[t.v[2]], g.y[t.v[2]]};
    const double t00 = a.x - c.x, t01 = b.x - c.x, t10 = a.y - c.y, t11 = b.y - c.y;
    const double det = t00 * t11 - t01 * t10, qx = q.x - c.x, qy = q.y - c.y;
    l[0] = (t11 * qx - t01 * qy) / det;
    l[1] = (t00 * qy - t10 * qx) / det;
    l[2] = 1.0 - l[0] - l[1];
    for (int k = 0; k < 3; ++k) v[k] = g.idx[t.v[k]];
    return true;
}

// ---- griddata(..., 'linear', fill_value=0) at the pixels whose value reaches the frame: interior pixels under
// the 9x9 mask, and the clamped neighbour of every masked pixel of the outermost ring.
__global__ void k_interp(pcd::Grid g, const int* __restrict__ count, const int* __restrict__ hull,
                         const int* __restrict__ hull_n, const uint8_t* __restrict__ m9,
                         const int* __restrict__ vidx, const float* __restrict__ colors, int W, int H,
                         double* __restrict__ interp, int* __restrict__ status) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    const int x = (int)(p % W), y = (int)(p / W);
    double out[3] = {0.0, 0.0, 0.0};
    bool need = false;
    if (!ring0(x, y, W, H)) {
        need = m9[p] != 0;
        for (int dy = -1; dy <= 1 && !need; ++dy)
            for (int dx = -1; dx <= 1 && !need; ++dx) {
                const int rx = x + dx, ry = y + dy;
                if (rx < 0 || ry < 0 || rx >= W || ry >= H || !ring0(rx, ry, W, H)) continue;
                const int tx = rx < 1 ? 1 : (rx > W - 2 ? W - 2 : rx), ty = ry < 1 ? 1 : (ry > H - 2 ? H - 2 : ry);
                need = tx == x && ty == y && m9[(int64_t)ry * W + rx] != 0;
            }
    }
    if (need) {
        int st = 0, v[3];
        double l[3];
        if (locate_linear(g, *count, hull, *hull_n, pcd::Pt{(double)x, (double)y}, v, l, st)) {
            for (int k = 0; k < 3; ++k) {
                const float* col = colors + (int64_t)vidx[v[k]] * 3;
                for (int ch = 0; ch < 3; ++ch) out[ch] = out[ch] + l[k] * (double)col[ch];
            }
        }
        if (st) atomicOr(status, st);
    }
    for (int ch = 0; ch < 3; ++ch) interp[p * 3 + ch] = out[ch];
}

// ---- the reference's expressions, one pixel at a time
// imagej = edgemask*imagej + (1-edgemask)*np.pad(imagej[1:-1,1:-1], 1, 'edge')
// imagej = maskj*imagej + (1-maskj)*(-1);   keep = imagej.sum(-1) != -3
__global__ void k_assemble(const double* __restrict__ interp, const uint8_t* __restrict__ m9, int W, int H,
                           double* __restrict__ img, uint8_t* __restrict__ keep) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    const int x = (int)(p % W), y = (int)(p / W);
    const double e = (x >= 2 && x <= W - 3 && y >= 2 && y <= H - 3) ? 1.0 : 0.0;
    const int tx = x < 1 ? 1 : (x > W - 2 ? W - 2 : x), ty = y < 1 ? 1 : (y > H - 2 ? H - 2 : y);
    const int64_t pp = (int64_t)ty * W + tx;
    const double m = m9[p] ? 1.0 : 0.0;
    const double fill = m9[p] ? -0.0 : -1.0;                           // (1 - maskj) * (-1) in float32
    double s = 0.0;
    for (int ch = 0; ch < 3; ++ch) {
        const double v1 = __dadd_rn(__dmul_rn(e, interp[p * 3 + ch]), __dmul_rn(1.0 - e, interp[pp * 3 + ch]));
        const double v2 = __dadd_rn(__dmul_rn(m, v1), fill);
        img[p * 3 + ch] = v2;
        s = ch == 0 ? v2 : __dadd_rn(s, v2);
    }
    keep[p] = s != -3.0;
}

// imagej = maskj*imagej + (1-maskj)*0, then np.round(imagej*255.).astype(np.uint8) or the float64 image
template <bool U8>
__global__ void k_finish(const double* __restrict__ img, const uint8_t* __restrict__ mask, int64_t npix,
                         uint8_t* __restrict__ frame, double* __restrict__ image, int32_t* __restrict__ mask_out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    const double m = mask[p] ? 1.0 : 0.0;
    for (int ch = 0; ch < 3; ++ch) {
        const double v = __dadd_rn(__dmul_rn(m, img[p * 3 + ch]), 0.0);
        if (U8) frame[p * 3 + ch] = (uint8_t)(int64_t)rint(__dmul_rn(v, 255.0));
        else image[p * 3 + ch] = v;
    }
    if (!U8) mask_out[p] = mask[p];
}

__global__ void k_copy_count(const int* __restrict__ count, int32_t* __restrict__ dst) { *dst = *count; }

// ---- scratch layout
struct Layout {
    size_t flags, pos, sums, count, vidx, cx, cy, rx, ry, cell_count, cell_start, cursor, cell_sums, sidx, sx, sy,
        mround, mtmp, m9, interp, img, keep, mask, ext, cand_count, cand_start, cand_sums, cand_n, cand,
        hull, hull_n, total;
};

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

Layout layout(int64_t n, int H, int W) {
    const GridDims g = grid_dims(n, H, W);
    const int64_t ncell = (int64_t)g.gw * g.gh, npix = (int64_t)H * W, nn = n > 0 ? n : 1;
    Layout L{};
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes); return at; };
    L.flags = take(4 * nn); L.pos = take(4 * nn);
    L.sums = take(4 * ((nn > ncell + 1 ? nn : ncell + 1) / SCAN_BLOCK + 1));
    L.count = take(4);
    L.vidx = take(4 * nn); L.cx = take(8 * nn); L.cy = take(8 * nn); L.rx = take(4 * nn); L.ry = take(4 * nn);
    L.cell_count = take(4 * (ncell + 1)); L.cell_start = take(4 * (ncell + 1)); L.cursor = take(4 * (ncell + 1));
    L.cell_sums = take(4 * ((ncell + 1) / SCAN_BLOCK + 1));
    L.sidx = take(4 * nn); L.sx = take(8 * nn); L.sy = take(8 * nn);
    L.mround = take(npix); L.mtmp = take(npix); L.m9 = take(npix);
    L.interp = take(24 * npix); L.img = take(24 * npix); L.keep = take(npix); L.mask = take(npix);
    L.ext = take(8 * ((int64_t)g.gw + g.gh));
    L.cand_count = take(4 * (ncell + 1)); L.cand_start = take(4 * (ncell + 1));
    L.cand_sums = take(4 * ((ncell + 1) / SCAN_BLOCK + 1)); L.cand_n = take(4);
    L.cand = take(4 * nn); L.hull = take(4 * (2 * nn + 1)); L.hull_n = take(4);
    L.total = o;
    return L;
}

bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

struct ViewOut {
    uint8_t* frame; double* image; int32_t* mask;                      // one of frame / (image, mask)
    int* vidx; double* cx; double* cy; int* rx; int* ry;               // compact outputs (scratch or caller's)
    int32_t* count_out;
};

// The buffers of one triangulation: the cell grid of the points, the hull candidates and the hull.
struct TriBufs {
    int *cell_count, *cell_start, *cursor, *cell_sums, *sidx;
    double *sx, *sy;
    int *ext, *cand_count, *cand_start, *cand_sums, *cand_n, *cand, *hull, *hull_n;
};

// Bins the first *count of the points (cx, cy) (at most n) into the cell grid gd, ascending index within a cell, and
// builds their convex hull: what locate_linear needs. Shared by the warp and the grow stage.
pcd::Grid enqueue_triangulate(const double* cx, const double* cy, const int* count, int64_t n, const GridDims& gd,
                              const TriBufs& b, int32_t* status, cudaStream_t st) {
    const int ncell = gd.gw * gd.gh;
    const int T = 256;
    const int nbp = (int)((n + T - 1) / T);
    cudaMemsetAsync(b.cell_count, 0, 4 * (size_t)(ncell + 1), st);
    if (n > 0) k_cell_count<<<nbp, T, 0, st>>>(cx, cy, count, gd, b.cell_count);
    exclusive_scan(b.cell_count, b.cell_start, ncell + 1, b.cell_sums, nullptr, st);
    if (n > 0) {
        cudaMemcpyAsync(b.cursor, b.cell_start, 4 * (size_t)ncell, cudaMemcpyDeviceToDevice, st);
        k_cell_scatter<<<nbp, T, 0, st>>>(cx, cy, count, gd, b.cursor, b.sidx);
        k_cell_sort<<<(ncell + T - 1) / T, T, 0, st>>>(b.cell_start, ncell, b.sidx);
        k_cell_gather<<<nbp, T, 0, st>>>(count, b.sidx, cx, cy, b.sx, b.sy);
    }
    int* top = b.ext; int* bot = top + gd.gw; int* left = bot + gd.gw; int* right = left + gd.gh;
    const int nbc = (ncell + T - 1) / T;
    cudaMemsetAsync(top, 0xff, 4 * (size_t)gd.gw, st);                // -1
    cudaMemsetAsync(bot, 0x7f, 4 * (size_t)gd.gw, st);                // larger than any row
    cudaMemsetAsync(left, 0x7f, 4 * (size_t)gd.gh, st);
    cudaMemsetAsync(right, 0xff, 4 * (size_t)gd.gh, st);
    cudaMemsetAsync(b.cand_count + ncell, 0, 4, st);
    k_extents<<<nbc, T, 0, st>>>(b.cell_start, gd.gw, gd.gh, top, bot, left, right);
    k_cand_count<<<nbc, T, 0, st>>>(b.cell_start, gd.gw, gd.gh, top, bot, left, right, b.cand_count);
    exclusive_scan(b.cand_count, b.cand_start, ncell + 1, b.cand_sums, b.cand_n, st);
    k_cand_gather<<<nbc, T, 0, st>>>(b.cell_start, gd.gw, gd.gh, b.cand_start, b.cand);
    k_cand_sort<<<(gd.gw + T - 1) / T, T, 0, st>>>(b.cand_start, gd.gw, gd.gh, b.sx, b.sy, b.sidx, b.cand);
    k_chain<<<1, 1, 0, st>>>(b.sx, b.sy, b.cand, b.cand_n, b.hull, b.hull_n, status);
    return pcd::Grid{gd.gw, gd.gh, gd.s, gd.inv_s, b.cell_start, b.sx, b.sy, b.sidx};
}

int enqueue_view(const double* pts, const float* colors, int64_t n, const Cam& cam, int H, int W, char* scratch,
                 const Layout& L, const ViewOut& o, int32_t* status, cudaStream_t st) {
    const GridDims gd = grid_dims(n, H, W);
    const int64_t npix = (int64_t)H * W;
    int* flags = (int*)(scratch + L.flags); int* pos = (int*)(scratch + L.pos); int* sums = (int*)(scratch + L.sums);
    int* count = (int*)(scratch + L.count);
    uint8_t* mround = (uint8_t*)(scratch + L.mround); uint8_t* mtmp = (uint8_t*)(scratch + L.mtmp);
    uint8_t* m9 = (uint8_t*)(scratch + L.m9);
    double* interp = (double*)(scratch + L.interp); double* img = (double*)(scratch + L.img);
    uint8_t* keep = (uint8_t*)(scratch + L.keep); uint8_t* mask = (uint8_t*)(scratch + L.mask);
    const TriBufs tb{(int*)(scratch + L.cell_count), (int*)(scratch + L.cell_start), (int*)(scratch + L.cursor),
                     (int*)(scratch + L.cell_sums), (int*)(scratch + L.sidx), (double*)(scratch + L.sx),
                     (double*)(scratch + L.sy), (int*)(scratch + L.ext), (int*)(scratch + L.cand_count),
                     (int*)(scratch + L.cand_start), (int*)(scratch + L.cand_sums), (int*)(scratch + L.cand_n),
                     (int*)(scratch + L.cand), (int*)(scratch + L.hull), (int*)(scratch + L.hull_n)};

    cudaMemsetAsync(mround, 0, npix, st);
    cudaMemsetAsync(count, 0, 4, st);
    const int T = 256;
    const int nbp = (int)((n + T - 1) / T);
    if (n > 0) {
        k_flags<<<nbp, T, 0, st>>>(pts, n, cam, W, H, flags);
        exclusive_scan(flags, pos, n, sums, count, st);
        k_compact<<<nbp, T, 0, st>>>(pts, n, cam, W, H, flags, pos, o.vidx, o.cx, o.cy, o.rx, o.ry, mround);
    }
    if (o.count_out) k_copy_count<<<1, 1, 0, st>>>(count, o.count_out);
    const int nbx = (int)((npix + T - 1) / T);
    k_filter<true, 4, true><<<nbx, T, 0, st>>>(mround, mtmp, W, H);
    k_filter<true, 4, false><<<nbx, T, 0, st>>>(mtmp, m9, W, H);
    const pcd::Grid g = enqueue_triangulate(o.cx, o.cy, count, n, gd, tb, status, st);
    k_interp<<<(int)((npix + 127) / 128), 128, 0, st>>>(g, count, tb.hull, tb.hull_n, m9, o.vidx, colors, W, H, interp,
                                                         status);
    k_assemble<<<nbx, T, 0, st>>>(interp, m9, W, H, img, keep);
    k_filter<false, 5, true><<<nbx, T, 0, st>>>(keep, mtmp, W, H);
    k_filter<false, 5, false><<<nbx, T, 0, st>>>(mtmp, mask, W, H);
    if (o.frame) k_finish<true><<<nbx, T, 0, st>>>(img, mask, npix, o.frame, nullptr, nullptr);
    else k_finish<false><<<nbx, T, 0, st>>>(img, mask, npix, nullptr, o.image, o.mask);
    return cudaPeekAtLastError() == cudaSuccess ? GSPCD_OK : GSPCD_ECUDA;
}

Cam make_cam(const double* pose, const double* K) {
    Cam c;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c.R[3 * i + j] = pose[3 * i + j];
    for (int i = 0; i < 3; ++i) c.T[i] = pose[9 + i];
    for (int i = 0; i < 9; ++i) c.K[i] = K[i];
    return c;
}

bool common_args_ok(const double* pts, const float* colors, int64_t n, const double* K, int H, int W,
                    int32_t* status, void* scratch, uint64_t scratch_bytes) {
    if (n < 0 || n > (int64_t)INT32_MAX / 2 || H < 3 || W < 3 || (int64_t)H * W > (int64_t)INT32_MAX / 4) return false;
    if (!K || !status || !scratch || !aligned(status, 4) || !aligned(scratch, 256)) return false;
    if (n > 0 && (!pts || !colors || !aligned(pts, 8) || !aligned(colors, 4))) return false;
    return scratch_bytes >= layout(n, H, W).total;
}

// ---- the grow stage (gspcd_grow_view): border points, their depth corrections, griddata linear / nearest over the
// inpainted pixels, back-projection. Every expression follows the reference's numpy / torch one, with the rounding
// of the CPU BLAS for a [3x3] @ [3xn] product: fma(a2, b2, fma(a1, b1, a0 * b0)) per row, zero entries included
// (they decide signed zeros).
struct GrowMats {
    float invK[9], invR32[9], invRT32[3], origin[3];                   // float32 quantities of the reference
    double invK64[9], invR[9], invRT[3], R[9], T[3];
};

__device__ __forceinline__ float chain32(const float* a, float b0, float b1, float b2) {
    return __fmaf_rn(a[2], b2, __fmaf_rn(a[1], b1, __fmul_rn(a[0], b0)));
}
__device__ __forceinline__ double chain64(const double* a, double b0, double b1, double b2) {
    return __fma_rn(a[2], b2, __fma_rn(a[1], b1, __dmul_rn(a[0], b0)));
}

// x86's default NaN, which numpy's invalid operations produce
__device__ __forceinline__ double nan64() { return __longlong_as_double((long long)0xFFF8000000000000ull); }
__device__ __forceinline__ float nan32() { return __int_as_float((int)0xFFC00000u); }

// matmul(eye(4), [p; 1])[:3] / [-1], the identity trans3d the scale fit leaves: each coordinate plus zeros (-0.0
// becomes +0.0), and 0 * inf or 0 * NaN makes a point with any non-finite coordinate NaN throughout.
__device__ __forceinline__ void identity3d(float p[3]) {
    const bool fin = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
    for (int r = 0; r < 3; ++r) p[r] = fin ? __fadd_rn(p[r], 0.0f) : nan32();
}
__device__ __forceinline__ void identity3d(double p[3]) {
    const bool fin = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
    for (int r = 0; r < 3; ++r) p[r] = fin ? __dadd_rn(p[r], 0.0) : nan64();
}

// mask_hf at (ry, rx): |m - m(below)| + |m - m(right)| >= 0.3, the last row and column padded from their neighbours
__global__ void k_border_flags(const int32_t* __restrict__ rnd, int64_t nv, const int32_t* __restrict__ mask2, int W,
                               int H, int* __restrict__ flags) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv) return;
    const int x = min(rnd[j], W - 2), y = min(rnd[nv + j], H - 2);
    const int32_t m = mask2[(int64_t)y * W + x];
    flags[j] = (m != mask2[(int64_t)(y + 1) * W + x] || m != mask2[(int64_t)y * W + x + 1]) ? 1 : 0;
}

// One border point: the torch float32 back-projection of its round pixel, the ray from the camera origin, the cloud
// point's projection onto it, and z(R comp + T) - z(R campixel + T). F32: the first view's float32 cloud.
template <bool F32>
__global__ void k_border_values(const void* __restrict__ pts_v, int64_t n, const int32_t* __restrict__ valid_idx,
                                const double* __restrict__ coords, const int32_t* __restrict__ rnd, int64_t nv,
                                const int* __restrict__ flags, const int* __restrict__ pos,
                                const float* __restrict__ depth, int W, GrowMats M, double* __restrict__ px,
                                double* __restrict__ py, double* __restrict__ val, int32_t* __restrict__ border_idx) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv || !flags[j]) return;
    const int rx = rnd[j], ry = rnd[nv + j];
    const float d = depth[(int64_t)ry * W + rx];
    const float X = __fmul_rn((float)rx, d), Y = __fmul_rn((float)ry, d);
    float cam[3], cp[3], vc[3];
    for (int r = 0; r < 3; ++r) cam[r] = chain32(M.invK + 3 * r, X, Y, d);
    for (int r = 0; r < 3; ++r) cp[r] = __fsub_rn(chain32(M.invR32 + 3 * r, cam[0], cam[1], cam[2]), M.invRT32[r]);
    identity3d(cp);
    for (int r = 0; r < 3; ++r) vc[r] = __fsub_rn(cp[r], M.origin[r]);
    const float den = __fadd_rn(__fadd_rn(__fmul_rn(vc[0], vc[0]), __fmul_rn(vc[1], vc[1])), __fmul_rn(vc[2], vc[2]));
    const int64_t i = valid_idx[j];
    double comp[3];
    if (F32) {
        const float* pts = (const float*)pts_v;
        float vp[3];
        for (int r = 0; r < 3; ++r) vp[r] = __fsub_rn(pts[r * n + i], M.origin[r]);
        const float num = __fadd_rn(__fadd_rn(__fmul_rn(vp[0], vc[0]), __fmul_rn(vp[1], vc[1])), __fmul_rn(vp[2], vc[2]));
        const float coeff = __fdiv_rn(num, den);
        for (int r = 0; r < 3; ++r) comp[r] = (double)__fadd_rn(M.origin[r], __fmul_rn(vc[r], coeff));
    } else {
        const double* pts = (const double*)pts_v;
        double vp[3];
        for (int r = 0; r < 3; ++r) vp[r] = __dsub_rn(pts[r * n + i], (double)M.origin[r]);
        const double num = __dadd_rn(__dadd_rn(__dmul_rn(vp[0], (double)vc[0]), __dmul_rn(vp[1], (double)vc[1])),
                                     __dmul_rn(vp[2], (double)vc[2]));
        const double coeff = __ddiv_rn(num, (double)den);
        for (int r = 0; r < 3; ++r) comp[r] = __dadd_rn((double)M.origin[r], __dmul_rn((double)vc[r], coeff));
    }
    const double zc = __dadd_rn(chain64(M.R + 6, comp[0], comp[1], comp[2]), M.T[2]);
    const double zh = __dadd_rn(chain64(M.R + 6, (double)cp[0], (double)cp[1], (double)cp[2]), M.T[2]);
    const int k = pos[j];
    px[k] = coords[j];
    py[k] = coords[nv + j];
    val[k] = __dsub_rn(zc, zh);
    if (border_idx) border_idx[k] = (int32_t)j;
}

// The four image corners with value 0 after the border points, in the reference's order.
__global__ void k_corners(const int* __restrict__ nb, int W, int H, double* __restrict__ px, double* __restrict__ py,
                          double* __restrict__ val, int* __restrict__ npts, int32_t* __restrict__ n_border) {
    const int b = *nb;
    const double cx[4] = {0.0, 0.0, (double)(W - 1), (double)(W - 1)}, cy[4] = {0.0, (double)(H - 1), 0.0, (double)(H - 1)};
    for (int k = 0; k < 4; ++k) { px[b + k] = cx[k]; py[b + k] = cy[k]; val[b + k] = 0.0; }
    *npts = b + 4;
    *n_border = b;
}

// np.where(1 - mask2): the pixels whose mask is not 1
__global__ void k_inpaint_flags(const int32_t* __restrict__ mask2, int64_t npix, int* __restrict__ flags) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < npix) flags[p] = mask2[p] != 1 ? 1 : 0;
}

// One inpainted pixel: griddata linear over the border points and corners (NaN outside the hull or from a NaN
// vertex value), nearest where that is NaN, then the back-projection of depth + correction and the colour.
__global__ void k_grow(pcd::Grid g, const int* __restrict__ npts, const int* __restrict__ hull,
                       const int* __restrict__ hull_n, const double* __restrict__ val,
                       const int32_t* __restrict__ mask2, const int* __restrict__ ipos, const float* __restrict__ depth,
                       const uint8_t* __restrict__ image, int W, int H, GrowMats M, int64_t m_new,
                       double* __restrict__ new_pts, float* __restrict__ new_colors, double* __restrict__ new_depth,
                       int* __restrict__ status) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H || mask2[p] == 1) return;
    const int64_t m = ipos[p];
    if (m >= m_new) return;
    const int x = (int)(p % W), y = (int)(p / W);
    const pcd::Pt q = {(double)x, (double)y};
    int st = 0, v[3];
    double l[3], nd = nan64();
    if (locate_linear(g, *npts, hull, *hull_n, q, v, l, st)) {
        nd = 0.0;
        for (int k = 0; k < 3; ++k) nd = nd + l[k] * val[v[k]];
    }
    if (isnan(nd)) {
        pcd::NearestQuery nq{&g, q, 0.0, -1, 0};
        pcd::NearestDone done{&nq};
        pcd::ring_search(g, q.x, q.y, nq, done);
        nd = val[g.idx[nq.best]];
    }
    if (st) atomicOr(status, st);
    const float d = depth[p];
    float pc[3];
    for (int r = 0; r < 3; ++r) pc[r] = chain32(M.invK + 3 * r, __fmul_rn((float)x, d), __fmul_rn((float)y, d), d);
    const double X = __dmul_rn((double)x, nd), Y = __dmul_rn((double)y, nd);
    double s[3], w[3];
    for (int r = 0; r < 3; ++r) s[r] = __dadd_rn((double)pc[r], chain64(M.invK64 + 3 * r, X, Y, nd));
    for (int r = 0; r < 3; ++r) w[r] = (double)__double2float_rn(__dsub_rn(chain64(M.invR + 3 * r, s[0], s[1], s[2]), M.invRT[r]));
    identity3d(w);
    for (int r = 0; r < 3; ++r) new_pts[r * m_new + m] = w[r];
    for (int ch = 0; ch < 3; ++ch) new_colors[m * 3 + ch] = __fdiv_rn((float)image[p * 3 + ch], 255.0f);
    if (new_depth) new_depth[m] = nd;
}

struct GrowLayout {
    size_t flags, pos, sums, nb, npts, px, py, val, iflags, ipos, isums;
    size_t cell_count, cell_start, cursor, cell_sums, sidx, sx, sy, ext, cand_count, cand_start, cand_sums, cand_n,
        cand, hull, hull_n, total;
};

// The grid is sized for a border of about four image perimeters; only the search time depends on it.
GridDims grow_grid(int64_t nv, int H, int W) {
    const int64_t per = 4 * ((int64_t)H + W);
    return grid_dims((nv < per ? nv : per) + 4, H, W);
}

GrowLayout grow_layout(int64_t nv, int H, int W) {
    const GridDims g = grow_grid(nv, H, W);
    const int64_t ncell = (int64_t)g.gw * g.gh, npix = (int64_t)H * W, nn = nv > 0 ? nv : 1, np4 = nv + 4;
    GrowLayout L{};
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes); return at; };
    L.flags = take(4 * nn); L.pos = take(4 * nn); L.sums = take(4 * (nn / SCAN_BLOCK + 1));
    L.nb = take(4); L.npts = take(4);
    L.px = take(8 * np4); L.py = take(8 * np4); L.val = take(8 * np4);
    L.iflags = take(4 * npix); L.ipos = take(4 * npix); L.isums = take(4 * (npix / SCAN_BLOCK + 1));
    L.cell_count = take(4 * (ncell + 1)); L.cell_start = take(4 * (ncell + 1)); L.cursor = take(4 * (ncell + 1));
    L.cell_sums = take(4 * ((ncell + 1) / SCAN_BLOCK + 1));
    L.sidx = take(4 * np4); L.sx = take(8 * np4); L.sy = take(8 * np4);
    L.ext = take(8 * ((int64_t)g.gw + g.gh));
    L.cand_count = take(4 * (ncell + 1)); L.cand_start = take(4 * (ncell + 1));
    L.cand_sums = take(4 * ((ncell + 1) / SCAN_BLOCK + 1)); L.cand_n = take(4);
    L.cand = take(4 * np4); L.hull = take(4 * (2 * np4 + 1)); L.hull_n = take(4);
    L.total = o;
    return L;
}

GrowMats grow_mats(const double* m) {
    GrowMats M;
    for (int i = 0; i < 9; ++i) { M.invK[i] = (float)m[i]; M.invK64[i] = (double)(float)m[i]; }
    for (int i = 0; i < 9; ++i) M.invR32[i] = (float)m[9 + i];
    for (int i = 0; i < 3; ++i) { M.invRT32[i] = (float)m[18 + i]; M.origin[i] = (float)m[21 + i]; }
    for (int i = 0; i < 9; ++i) M.invR[i] = m[24 + i];
    for (int i = 0; i < 3; ++i) M.invRT[i] = m[33 + i];
    for (int i = 0; i < 9; ++i) M.R[i] = m[36 + i];
    for (int i = 0; i < 3; ++i) M.T[i] = m[45 + i];
    return M;
}

bool grow_sizes_ok(int64_t nv, int H, int W) {
    return nv >= 0 && nv <= (int64_t)INT32_MAX / 2 && H >= 3 && W >= 3 && (int64_t)H * W <= (int64_t)INT32_MAX / 4;
}

}  // namespace

extern "C" {

int gspcd_abi_version(void) { return 1; }

int gspcd_scratch_bytes(int64_t n, int32_t H, int32_t W, uint64_t* bytes) {
    if (!bytes || n < 0 || n > (int64_t)INT32_MAX / 2 || H < 3 || W < 3 || (int64_t)H * W > (int64_t)INT32_MAX / 4)
        return GSPCD_EINVAL;
    *bytes = layout(n, H, W).total;
    return GSPCD_OK;
}

int gspcd_align(const double* pts, const float* colors, int64_t n, const double* poses, const double* K,
                int32_t n_views, int32_t H, int32_t W, uint8_t* frames, int32_t* counts, int32_t* status,
                void* scratch, uint64_t scratch_bytes, void* stream) {
    if (!common_args_ok(pts, colors, n, K, H, W, status, scratch, scratch_bytes)) return GSPCD_EINVAL;
    if (n_views < 0 || (n_views > 0 && (!poses || !frames || !counts || !aligned(counts, 4)))) return GSPCD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const Layout L = layout(n, H, W);
    char* s = (char*)scratch;
    if (cudaMemsetAsync(status, 0, 4, st) != cudaSuccess) return GSPCD_ECUDA;
    const int64_t frame_bytes = (int64_t)H * W * 3;
    for (int v = 0; v < n_views; ++v) {
        ViewOut o{frames + v * frame_bytes, nullptr, nullptr, (int*)(s + L.vidx), (double*)(s + L.cx),
                  (double*)(s + L.cy), (int*)(s + L.rx), (int*)(s + L.ry), counts + v};
        const int rc = enqueue_view(pts, colors, n, make_cam(poses + 12 * v, K), H, W, s, L, o, status, st);
        if (rc) return rc;
    }
    return GSPCD_OK;
}

int gspcd_warp_view(const double* pts, const float* colors, int64_t n, const double* pose, const double* K,
                    int32_t H, int32_t W, double* image, int32_t* mask, int32_t* valid_idx, double* coords,
                    int32_t* round_coords, int32_t* count, int32_t* status, void* scratch, uint64_t scratch_bytes,
                    void* stream) {
    if (!common_args_ok(pts, colors, n, K, H, W, status, scratch, scratch_bytes)) return GSPCD_EINVAL;
    if (!pose || !image || !mask || !count || !aligned(image, 8) || !aligned(mask, 4) || !aligned(count, 4))
        return GSPCD_EINVAL;
    if (n > 0 && (!valid_idx || !coords || !round_coords || !aligned(valid_idx, 4) || !aligned(coords, 8) ||
                  !aligned(round_coords, 4)))
        return GSPCD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const Layout L = layout(n, H, W);
    char* s = (char*)scratch;
    if (cudaMemsetAsync(status, 0, 4, st) != cudaSuccess) return GSPCD_ECUDA;
    const int64_t nn = n > 0 ? n : 0;
    ViewOut o{nullptr, image, mask,
              n > 0 ? valid_idx : (int*)(s + L.vidx), n > 0 ? coords : (double*)(s + L.cx),
              n > 0 ? coords + nn : (double*)(s + L.cy), n > 0 ? round_coords : (int*)(s + L.rx),
              n > 0 ? round_coords + nn : (int*)(s + L.ry), count};
    return enqueue_view(pts, colors, n, make_cam(pose, K), H, W, s, L, o, status, st);
}

int gspcd_grow_scratch_bytes(int64_t n_valid, int32_t H, int32_t W, uint64_t* bytes) {
    if (!bytes || !grow_sizes_ok(n_valid, H, W)) return GSPCD_EINVAL;
    *bytes = grow_layout(n_valid, H, W).total;
    return GSPCD_OK;
}

int gspcd_grow_view(const void* pts, int64_t n, int32_t cloud_is_f32, const int32_t* valid_idx, const double* coords,
                    const int32_t* round_coords, int64_t n_valid, const int32_t* mask2, const float* depth,
                    const uint8_t* image, int32_t H, int32_t W, const double* mats, int64_t m_new, double* new_pts,
                    float* new_colors, double* new_depth, int32_t* border_idx, int32_t* n_border, int32_t* status,
                    void* scratch, uint64_t scratch_bytes, void* stream) {
    if (!grow_sizes_ok(n_valid, H, W) || n < n_valid || n > (int64_t)INT32_MAX / 2) return GSPCD_EINVAL;
    if (cloud_is_f32 != 0 && cloud_is_f32 != 1) return GSPCD_EINVAL;
    if (m_new < 0 || m_new > (int64_t)H * W) return GSPCD_EINVAL;
    if (!mask2 || !depth || !image || !mats || !new_pts || !new_colors || !n_border || !status || !scratch)
        return GSPCD_EINVAL;
    if (!aligned(mask2, 4) || !aligned(depth, 4) || !aligned(new_pts, 8) || !aligned(new_colors, 4) ||
        !aligned(n_border, 4) || !aligned(status, 4) || !aligned(scratch, 256))
        return GSPCD_EINVAL;
    if ((new_depth && !aligned(new_depth, 8)) || (border_idx && !aligned(border_idx, 4))) return GSPCD_EINVAL;
    if (n_valid > 0 && (!pts || !valid_idx || !coords || !round_coords || !aligned(pts, cloud_is_f32 ? 4 : 8) ||
                        !aligned(valid_idx, 4) || !aligned(coords, 8) || !aligned(round_coords, 4)))
        return GSPCD_EINVAL;
    const GrowLayout L = grow_layout(n_valid, H, W);
    if (scratch_bytes < L.total) return GSPCD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    char* s = (char*)scratch;
    const GrowMats M = grow_mats(mats);
    const GridDims gd = grow_grid(n_valid, H, W);
    const int64_t npix = (int64_t)H * W;
    int* flags = (int*)(s + L.flags); int* pos = (int*)(s + L.pos); int* nb = (int*)(s + L.nb);
    int* npts = (int*)(s + L.npts); int* ipos = (int*)(s + L.ipos); int* iflags = (int*)(s + L.iflags);
    double* px = (double*)(s + L.px); double* py = (double*)(s + L.py); double* val = (double*)(s + L.val);
    const TriBufs tb{(int*)(s + L.cell_count), (int*)(s + L.cell_start), (int*)(s + L.cursor), (int*)(s + L.cell_sums),
                     (int*)(s + L.sidx), (double*)(s + L.sx), (double*)(s + L.sy), (int*)(s + L.ext),
                     (int*)(s + L.cand_count), (int*)(s + L.cand_start), (int*)(s + L.cand_sums), (int*)(s + L.cand_n),
                     (int*)(s + L.cand), (int*)(s + L.hull), (int*)(s + L.hull_n)};
    if (cudaMemsetAsync(status, 0, 4, st) != cudaSuccess) return GSPCD_ECUDA;
    cudaMemsetAsync(nb, 0, 4, st);
    const int T = 256;
    const int nbv = (int)((n_valid + T - 1) / T);
    if (n_valid > 0) {
        k_border_flags<<<nbv, T, 0, st>>>(round_coords, n_valid, mask2, W, H, flags);
        exclusive_scan(flags, pos, n_valid, (int*)(s + L.sums), nb, st);
        if (cloud_is_f32)
            k_border_values<true><<<nbv, T, 0, st>>>(pts, n, valid_idx, coords, round_coords, n_valid, flags, pos, depth,
                                                     W, M, px, py, val, border_idx);
        else
            k_border_values<false><<<nbv, T, 0, st>>>(pts, n, valid_idx, coords, round_coords, n_valid, flags, pos,
                                                      depth, W, M, px, py, val, border_idx);
    }
    k_corners<<<1, 1, 0, st>>>(nb, W, H, px, py, val, npts, n_border);
    const int nbx = (int)((npix + T - 1) / T);
    k_inpaint_flags<<<nbx, T, 0, st>>>(mask2, npix, iflags);
    exclusive_scan(iflags, ipos, npix, (int*)(s + L.isums), nullptr, st);
    const pcd::Grid g = enqueue_triangulate(px, py, npts, n_valid + 4, gd, tb, status, st);
    k_grow<<<(int)((npix + 127) / 128), 128, 0, st>>>(g, npts, tb.hull, tb.hull_n, val, mask2, ipos, depth, image, W, H,
                                                       M, m_new, new_pts, new_colors, new_depth, status);
    return cudaPeekAtLastError() == cudaSuccess ? GSPCD_OK : GSPCD_ECUDA;
}

}  // extern "C"
