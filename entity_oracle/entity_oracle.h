/*
 * entity_oracle.h -- CPU ORACLE of bgs_render_entities (include/bgs.h).  TEST INFRASTRUCTURE ONLY: only tests/ and
 * scripts/ may load it.
 *
 * scene4d_oracle/'s joint frame with each cloud drawn with its own settings: cloud j's gaussians take global indices
 * o_j + i, are keyed on their base positions with their own uniform and sorted stably over (key, global index).  The
 * record of each is the one scene4d_oracle/ writes for it with settings[j] as the frame's (num_classes[j] for a 4D
 * Classification entity; a non-4D entity in Velocity is undrawn; Depth colours from the joint sorted[1] / sorted[N-1]),
 * in bgs_debug_projected's layout with its own entity's aabb.  Binning is the oracle's; the tile walk decides each
 * (pixel, splat) pair with that splat's own entity's coverage rule (quad-uv, conic or surfel), in joint order, depth-tested
 * against `scene` when given.  Non-4D entities in Classification or OpticalFlow are not covered (returns 3).  With every
 * entity's settings equal this is s4o_frame, bit for bit.  FP policy: oracle/bgs_oracle.h's.
 */
#ifndef ENTITY_ORACLE_H
#define ENTITY_ORACLE_H
#include <stdint.h>

#include "../scene4d_oracle/scene4d_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* s4o_frame's arguments and outputs, with settings[j] and num_classes[j] per cloud (radix_sort_depth_bits: entity 0's). */
int eo_frame(uint32_t k, const s4o_cloud* clouds, const orc_view* view, const orc_settings* settings, const uint32_t* num_classes,
             const tor_temporal* ex, const float* scene, uint64_t pitch_bytes, uint32_t* n_vis, uint64_t* n_pairs, uint32_t* sorted,
             float* records, uint32_t* rank_to_id, float* depths, uint32_t* tile_ranges, uint32_t* tile_entries, uint64_t cap,
             float* image, int threads);

#ifdef __cplusplus
}
#endif
#endif
