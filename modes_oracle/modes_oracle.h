/*
 * modes_oracle.h -- CPU ORACLE of RasterizeMode::Classification and RasterizeMode::OpticalFlow's colour sources
 * (gaussian.wgsl:312-421, material/classification.wgsl:9-27, material/optical_flow.wgsl:16-53).  TEST INFRASTRUCTURE
 * ONLY: the product never links, loads or calls it.
 *
 * Both modes change only a splat's colour, so the rest of a record (geometry, opacity, bbox) is oracle/'s Color-mode
 * record; modes_oracle.py composes the two.  FP policy as oracle/bgs_oracle.h: IEEE binary32, round to nearest even,
 * no contraction (-ffp-contract=off), every step in the order include/bgs.h ("The rule, exactly") writes it; min / max
 * ignore a NaN operand; atan2 is the fixed f64 series restated below, the same as csrc/project.cu's det_atan2.
 */
#ifndef MODES_ORACLE_H
#define MODES_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* bevy_render::color_operations::hsv_to_rgb per element: rgb_out = n * 3 floats */
void mo_hsv_to_rgb(uint32_t n, const float* h, const float* s, const float* v, float* rgb_out);
/* the fixed-series atan2 (y, x) per element */
void mo_atan2(uint32_t n, const float* y, const float* x, float* out);
/* Classification: sh_rgb (n * 3, the Color-mode colour), vis (n) -> rgb_out (n * 3); num_classes > 0 */
void mo_class_colour(uint32_t n, const float* sh_rgb, const float* vis, uint32_t num_classes, float* rgb_out);
/* OpticalFlow: pos (n * 4: x, y, z, visibility), model / clip / prev_clip column-major -> rgb_out (n * 3) */
void mo_flow_colour(uint32_t n, const float* pos, const float* model, const float* clip, const float* prev_clip,
                    float delta_time, float* rgb_out);

#ifdef __cplusplus
}
#endif
#endif
