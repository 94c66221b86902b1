/* Point-cloud warp for LucidDreamer's scene generation, on the device (sm_90a).
 *
 * Warps a coloured point cloud into camera views the way LucidDreamer.generate_pcd does with
 * scipy.interpolate.griddata(..., method='linear', fill_value=0): project, round mask, linear interpolation in the
 * Delaunay triangulation of the projected points, edge ring, 9x9 maximum and 11x11 minimum filters (reflect).
 *
 * gspcd_grow_view grows the cloud from an inpainted view: border depth compensation, Delaunay-linear interpolation
 * and back-projection.
 *
 * Conventions: every array argument is device memory except `poses`, `K` and `mats`, which are host arrays read
 * during the call. pts is [3, N] float64 (rows x, y, z), colors [N, 3] float32. A pose is 12 float64: R row-major, then T.
 * Work is enqueued on `stream` (a cudaStream_t, 0 = legacy default) without host synchronisation; results are
 * valid once the stream reaches them. `status` receives 0, or a nonzero code when an exact predicate needed more
 * precision than it carries or a walk exceeded its step cap; the output is then not to be trusted.
 * Functions return 0 or a negative error code. Scratch is caller-provided, 256-byte aligned.
 */
#ifndef GSPCD_H
#define GSPCD_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSPCD_OK 0
#define GSPCD_EINVAL (-22)
#define GSPCD_ECUDA (-5)

int gspcd_abi_version(void);

/* Scratch needed by gspcd_align and gspcd_warp_view for N points and an H x W view (W, H >= 3). */
int gspcd_scratch_bytes(int64_t n, int32_t H, int32_t W, uint64_t *bytes);

/* All n_views views of one alignment. frames: [n_views, H, W, 3] uint8 = round(image * 255);
 * counts: [n_views] int32, the number of valid (projected in-view) points of each view. */
int gspcd_align(const double *pts, const float *colors, int64_t n, const double *poses, const double *K,
                int32_t n_views, int32_t H, int32_t W, uint8_t *frames, int32_t *counts, int32_t *status,
                void *scratch, uint64_t scratch_bytes, void *stream);

/* One dreaming-stage view. image: [H, W, 3] float64; mask: [H, W] int32 (0/1); valid_idx: [N] int32, the first
 * count[0] entries are the valid point indices, ascending; coords: [2, N] float64 and round_coords: [2, N] int32,
 * the first count[0] columns of each row used. */
int gspcd_warp_view(const double *pts, const float *colors, int64_t n, const double *pose, const double *K,
                    int32_t H, int32_t W, double *image, int32_t *mask, int32_t *valid_idx, double *coords,
                    int32_t *round_coords, int32_t *count, int32_t *status, void *scratch, uint64_t scratch_bytes,
                    void *stream);

/* Scratch needed by gspcd_grow_view for n_valid valid points and an H x W view (W, H >= 3). */
int gspcd_grow_scratch_bytes(int64_t n_valid, int32_t H, int32_t W, uint64_t *bytes);

/* One dreaming-stage growth of the cloud from its inpainted view (generate_pcd after the depth model): the valid
 * points whose round pixel lies on the border of mask2 (|m - m(below)| + |m - m(right)| >= 0.3, last row and column
 * padded), the depth correction of each along its camera ray, griddata linear over them and the four image corners
 * (value 0) at the pixels where mask2 != 1, in row-major order, griddata nearest where linear is NaN, and the
 * back-projection of depth + correction into world space. The reference's scale fit is not run: it leaves trans3d
 * the identity, whose only effect is -0.0 -> +0.0 and NaN for a point with a non-finite coordinate.
 *
 * pts: [3, n], float32 when cloud_is_f32 (the first view's cloud) else float64; valid_idx [n_valid] int32, coords
 * [2, n_valid] float64, round_coords [2, n_valid] int32: gspcd_warp_view's outputs; mask2 [H, W] int32; depth
 * [H, W] float32; image [H, W, 3] uint8. mats: 48 host float64, the caller's numpy / torch results: inv(K) as float32
 * (9), float32(inv(R)) (9), its torch product with float32(T) (3), -float32(inv(R).dot(T)) (3), inv(R) (9),
 * inv(R).dot(T) (3), R (9), T (3), matrices row-major. m_new: the number of pixels with mask2 != 1.
 * Out: new_pts [3, m_new] float64, new_colors [m_new, 3] float32 (= image / 255.f), and, when not NULL, new_depth
 * [m_new] float64 (the interpolated correction) and border_idx [n_valid] int32 (its first n_border[0] entries: the
 * positions in valid_idx of the border points, ascending). Nearest ties go to the lowest index (border points in
 * order, then the corners); scipy's cKDTree does not pin its tie order. 3x3 products round as
 * fma(a2, b2, fma(a1, b1, a0 * b0)), which is what numpy's and torch's CPU BLAS do for two or more columns. */
int gspcd_grow_view(const void *pts, int64_t n, int32_t cloud_is_f32, const int32_t *valid_idx, const double *coords,
                    const int32_t *round_coords, int64_t n_valid, const int32_t *mask2, const float *depth,
                    const uint8_t *image, int32_t H, int32_t W, const double *mats, int64_t m_new, double *new_pts,
                    float *new_colors, double *new_depth, int32_t *border_idx, int32_t *n_border, int32_t *status,
                    void *scratch, uint64_t scratch_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif
