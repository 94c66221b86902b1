/* Point-cloud warp for LucidDreamer's scene generation, on the device (sm_90a).
 *
 * Warps a coloured point cloud into camera views the way LucidDreamer.generate_pcd does with
 * scipy.interpolate.griddata(..., method='linear', fill_value=0): project, round mask, linear interpolation in the
 * Delaunay triangulation of the projected points, edge ring, 9x9 maximum and 11x11 minimum filters (reflect).
 *
 * Conventions: every array argument is device memory except `poses` and `K`, which are host arrays read during
 * the call. pts is [3, N] float64 (rows x, y, z), colors [N, 3] float32. A pose is 12 float64: R row-major, then T.
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

#ifdef __cplusplus
}
#endif
#endif
