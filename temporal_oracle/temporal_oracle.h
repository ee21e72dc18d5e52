/*
 * temporal_oracle.h -- CPU ORACLE of bgs_render_4d (include/bgs.h: the conditioning of a Gaussian4d on time, its record,
 * spherindrical colour and Velocity, and the tile walk of a frame).  TEST INFRASTRUCTURE ONLY: the product never links,
 * loads or calls it.
 *
 * Key-gen, the sort, binning and the coverage decision are oracle/bgs_oracle.cpp's (compiled into this library); the
 * hue and atan2 of Classification / OpticalFlow are modes_oracle/'s.  FP policy as oracle/bgs_oracle.h: IEEE binary32,
 * round to nearest even, no contraction, every step in the order include/bgs.h writes it; exp and cos are the fixed f64
 * series restated below, the same as csrc/project_math.cuh's det_exp / det_cos.  The SH sums are evaluated unfused
 * (the GPU fuses them: those colours are compared under a bound).
 */
#ifndef TEMPORAL_ORACLE_H
#define TEMPORAL_ORACLE_H
#include <stdint.h>

#include "../oracle/bgs_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* bgs_render_4d's time window and extras */
typedef struct {
    float time_start, time_stop;
    float prev_clip_from_world[16];
    float delta_time;
    uint32_t num_classes;
} tor_temporal;

void tor_exp(uint32_t n, const float* x, float* out);
void tor_cos(uint32_t n, const float* x, float* out);
/* the conditioning of each gaussian at time t: cov6 (n*6), delta_mean (n*3), marginal (n), mask (n) */
void tor_condition(uint32_t n, const float* rot8, const float* so, const float* tt, float global_scale, float t, float* cov6,
                   float* delta_mean, float* marginal, uint8_t* mask);
/* One frame: n_vis and, when the arrays are non-NULL, the records by front-to-back rank (12 floats each, the layout of
 * bgs_debug_projected), rank -> gaussian index, the splat depths d by rank, and the tile-mode image (W*H*4, over opaque
 * black) depth-tested against `scene` (NULL: no test).  Call once with NULL arrays for n_vis. */
int tor_frame(uint32_t n, const float* pos_vis, const float* sh144, const float* rot8, const float* so, const float* tt,
              const orc_view* view, const orc_uniform* u, const orc_settings* s, const tor_temporal* tp, const float* scene,
              uint64_t pitch_bytes, uint32_t* n_vis, float* records, uint32_t* rank_to_id, float* depths, float* image,
              int threads);

#ifdef __cplusplus
}
#endif
#endif
