/* Training-scene images for LucidDreamer's Scene, on the device (sm_90a).
 *
 * For every frame of a scene, gsscene_camera_images makes the two images a training camera carries:
 *   original_image  the frame composited over a black or white background as the reference's loadCamerasFromData
 *                   does it: norm = u / 255.0 and rgb * a + bg * (1 - a) in float64, rounded to float32, clamped to
 *                   [0, 1];
 *   canny_mask      1 - cv2.Canny(u8, 50, 150) / 255 with u8 = (uint8)(original_image * 255.f), as image2canny makes
 *                   it: OpenCV's Canny for 8-bit three-channel input, aperture 3, L1 norm. 3x3 Sobel per channel with
 *                   replicated borders, the channel with the largest |dx| + |dy| (ties to the lowest), non-maximum
 *                   suppression with OpenCV's integer tan 22.5 deg sectors and its `>` / `>=` neighbour tests,
 *                   thresholds m > 50 and m > 150, and hysteresis as the 8-connected closure of the strong pixels
 *                   through the candidates (union-find over the candidate pixels; integer atomics only, so the result
 *                   does not depend on scheduling).
 *
 * Conventions: every array argument is device memory. Work is enqueued on `stream` (a cudaStream_t, 0 = legacy
 * default) as a fixed sequence of launches, without host synchronisation, so a call can be captured in a CUDA graph.
 * Functions return 0 or a negative error code. Scratch is caller-provided, 256-byte aligned.
 */
#ifndef GSSCENE_H
#define GSSCENE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSSCENE_OK 0
#define GSSCENE_EINVAL (-22)
#define GSSCENE_ECUDA (-5)

int gsscene_abi_version(void);

/* Scratch needed by gsscene_camera_images for F frames of H x W (F >= 0, H, W >= 1, F * H * W < 2^31). */
int gsscene_scratch_bytes(int32_t F, int32_t H, int32_t W, uint64_t *bytes);

/* All F frames of a scene in one call. frames: [F, H, W, C] uint8 with C = 3 (alpha 255) or 4 (RGBA);
 * white_background: 0 (black) or 1 (white). Out: image [F, 3, H, W] float32, canny_mask [F, H, W] float32. */
int gsscene_camera_images(const uint8_t *frames, int32_t F, int32_t H, int32_t W, int32_t C, int32_t white_background,
                          float *image, float *canny_mask, void *scratch, uint64_t scratch_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif
