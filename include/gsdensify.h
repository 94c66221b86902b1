/* Densification and pruning of a Gaussian model on the device (sm_90a), as the reference GaussianModel's
 * densify_and_prune and reset_opacity compute them, bit for bit.
 *
 * A densify is three calls around one random draw the caller makes with torch's generator:
 *
 *   gsdensify_plan    per row of the current model: clone, split and the final prune decisions, and the exclusive
 *                     offsets of every output row. Writes counts[4] = {clones, splits, surviving originals, new P}
 *                     to device memory: the one thing the host reads.
 *   gsdensify_map     the output row list [surviving originals, clones, split copy 1, split copy 2] with pruned rows
 *                     left out: map[o] = {source row, kind}, kind = -2 original, -1 clone, k >= 0 split sample row k
 *                     (k < S: copy 1, k >= S: copy 2). Also writes stds [2S, 3] = exp(scaling) of the split rows,
 *                     repeated twice, the std of the caller's torch.normal(mean=zeros, std=stds).
 *   gsdensify_apply   one gather over every output tensor along the map (parameters, Adam moments), split rows'
 *                     xyz = R(rotation) @ sample + xyz and scaling = log(exp(s) * float32(1 / 1.6)).
 *
 * gsdensify_reset_opacity is one launch: log(x / (1 - x)) with x = min(sigmoid(o), 0.01f), and zero moments.
 *
 * The plan's thresholds are the reference's Python scalars cast to float32, as torch casts them:
 *   max_grad            clone: |g| >= max_grad, split: g >= max_grad, g = accum / denom with NaN -> 0
 *   dense_scale         float32(percent_dense * extent): clone when max(exp(s)) <= it, split when > it
 *   min_opacity         prune when sigmoid(o) < it
 *   screen              1 when the reference's `if max_screen_size:` holds; then also prune when
 *                       0 > max_screen (the statistics are zero by then) or max(exp(s)) > world_scale
 *   world_scale         float32(0.1 * extent)
 *
 * Conventions: every array argument is device memory, float32 rows contiguous. Work is enqueued on `stream`
 * (a cudaStream_t, 0 = legacy default) without host synchronisation. Functions return 0 or a negative error code.
 * Scratch is caller-provided, 256-byte aligned, and carries the plan to the map.
 */
#ifndef GSDENSIFY_H
#define GSDENSIFY_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSDENSIFY_OK 0
#define GSDENSIFY_EINVAL (-22)
#define GSDENSIFY_ECUDA (-5)

/* gsdensify_tensor.kind */
#define GSDENSIFY_PARAM 0      /* gathered for every output row */
#define GSDENSIFY_XYZ 1        /* gathered; split rows R(rotation) @ sample + xyz */
#define GSDENSIFY_SCALING 2    /* gathered; split rows log(exp(s) * float32(1 / 1.6)) */
#define GSDENSIFY_MOMENT 3     /* gathered for surviving originals, zero for clones and split copies */
#define GSDENSIFY_MAX_TENSORS 32

typedef struct {
    const float *src;          /* [P, width] */
    float *dst;                /* [P_new, width] */
    int32_t width;             /* floats per row, >= 1 */
    int32_t kind;
} gsdensify_tensor;

int gsdensify_abi_version(void);

/* Scratch needed by gsdensify_plan / gsdensify_map for a model of P rows (0 <= P < 2^30). */
int gsdensify_scratch_bytes(int32_t P, uint64_t *bytes);

/* accum, denom, opacity: [P, 1]; scaling: [P, 3]; counts: int32[4] in device memory. */
int gsdensify_plan(int32_t P, const float *accum, const float *denom, const float *scaling, const float *opacity,
                   float max_grad, float dense_scale, float min_opacity, int32_t screen, float max_screen,
                   float world_scale, int32_t *counts, void *scratch, uint64_t scratch_bytes, void *stream);

/* After gsdensify_plan on the same scratch: S and P_new are counts[1] and counts[3]. map: int32[P_new, 2],
 * stds: [2S, 3]. */
int gsdensify_map(int32_t P, const float *scaling, int32_t S, int32_t P_new, int32_t *map, float *stds, void *scratch,
                  uint64_t scratch_bytes, void *stream);

/* tensors: host array of n descriptors. rotation: [P, 4] source rotations, samples: [2S, 3] (read for split rows'
 * xyz; the 2S products are rounded as torch.bmm rounds a batch of 2S). Every dst has P_new rows;
 * P_new * width < 2^31. */
int gsdensify_apply(const int32_t *map, int32_t P_new, const gsdensify_tensor *tensors, int32_t n,
                    const float *rotation, const float *samples, int32_t S, void *stream);

/* opacity: [P, 1] in; out, exp_avg, exp_avg_sq: [P, 1] out (exp_avg / exp_avg_sq may be null: not written). */
int gsdensify_reset_opacity(int32_t P, const float *opacity, float *out, float *exp_avg, float *exp_avg_sq,
                            void *stream);

#ifdef __cplusplus
}
#endif
#endif
