/*
 * scene4d_oracle.h -- CPU ORACLE of bgs_render_scene_4d (include/bgs.h).  TEST INFRASTRUCTURE ONLY: only tests/ and
 * scripts/ may load it.
 *
 * scene_oracle/'s joint frame with Gaussian4d clouds among the k: cloud j's gaussians take global indices o_j + i; every
 * gaussian is keyed by the oracle on its base position with its own cloud's uniform; the depth sort is stable over (key,
 * global index); the Depth range is sorted[1] / sorted[N-1] of that joint list (base positions).  A 3D gaussian's record
 * is oracle/'s (the Depth colour filled from the joint range, as scene_oracle/ does); in a Velocity frame it is the
 * undrawn record.  A 4D gaussian's record and splat depth are temporal_oracle/'s per-gaussian rule at its cloud's
 * uniform time and window.  Binning and the tile walk (depth-tested against `scene` when given) then run on the joint
 * record set.  FP policy: oracle/bgs_oracle.h's (temporal_oracle.cpp is compiled into this library).
 */
#ifndef SCENE4D_ORACLE_H
#define SCENE4D_ORACLE_H
#include <stdint.h>

#include "../oracle/bgs_oracle.h"
#include "../temporal_oracle/temporal_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* One listed cloud.  kind 0: a 3D cloud as scene_oracle/ reads it (sh 48 floats and rot 4 per gaussian, cov_pre: its
 * planes hold decoded covariance records); kind 1: a Gaussian4d cloud (sh 144, rot 8, tt 4 per gaussian; its time is
 * u.time, its window [time_start, time_stop]). */
typedef struct {
    uint32_t n;
    uint32_t kind;
    uint32_t cov_pre;
    const float* pos_vis;
    const float* sh;
    const float* rot;
    const float* scale_opacity;
    const float* tt;
    orc_uniform u;
    float time_start, time_stop;
} s4o_cloud;

/* One frame.  s: the frame's settings (gaussian_mode the 3D clouds'; 4D clouds are projected as Gaussian4d); ex: the
 * extras (its time window is not read).  n_vis and n_pairs always; when non-NULL: sorted (N * 2: key, global index),
 * records (n_vis * 12, bgs_debug_projected's layout by front-to-back rank), rank_to_id, depths (splat depths by rank),
 * tile_ranges (T * 2), tile_entries (up to cap) and image (W * H * 4, the tile walk over opaque black, depth-tested
 * against `scene` unless it is NULL).  Call once with NULL arrays for the sizes. */
int s4o_frame(uint32_t k, const s4o_cloud* clouds, const orc_view* view, const orc_settings* s, const tor_temporal* ex,
              const float* scene, uint64_t pitch_bytes, uint32_t* n_vis, uint64_t* n_pairs, uint32_t* sorted, float* records,
              uint32_t* rank_to_id, float* depths, uint32_t* tile_ranges, uint32_t* tile_entries, uint64_t cap, float* image,
              int threads);

#ifdef __cplusplus
}
#endif
#endif
