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

/* eo_frame with each entity's flags (bgs_render_entities_ex): entity_flags[j] bit 0 (BGS_ENTITY_VISUALIZE_BOUNDING_BOX)
 * draws entity j's bounding boxes (include/bgs.h's BGS_FLAG_VISUALIZE_BOUNDING_BOX rule: a covered, depth-passing pair on
 * its quad's edge band blends (0.3, 1, 0.1) at alpha 1 and stops the pixel); entity_flags == NULL is eo_frame.  edge_mask
 * (W*H bytes, optional): 1 where an edge pair blended.  surfel_extra (16 floats per rank, optional): a 2DGS aabb rank's
 * surfel extras as the blend kernels stage them, e0 = (Rq, mean x, mean y, W / H), e1, e2, e3 = (T0, 0), (T1, 0),
 * (T2, 0) (gaussian_2d.wgsl's homography rows); zeros for the other ranks. */
int eo_frame_ex(uint32_t k, const s4o_cloud* clouds, const orc_view* view, const orc_settings* settings, const uint32_t* num_classes,
                const uint32_t* entity_flags, const tor_temporal* ex, const float* scene, uint64_t pitch_bytes, uint32_t* n_vis,
                uint64_t* n_pairs, uint32_t* sorted, float* records, uint32_t* rank_to_id, float* depths, uint32_t* tile_ranges,
                uint32_t* tile_entries, uint64_t cap, float* image, uint8_t* edge_mask, float* surfel_extra, int threads);

/* The overlay's edge decision per pair: splat record splats[j] (orc_splat, the oracle's own) at the pixel centre
 * (pixel_xy[2j], pixel_xy[2j+1]) under settings s (aabb, gaussian_mode as the blend reads them: 1 = conic, 0 = surfel).
 * covered[j]: the coverage decision (oracle/bgs_oracle.cpp's decide()); edge[j]: covered and on the edge band; s_xy
 * (optional, 2 per pair): s = uv * 0.5 + 0.5 of covered pairs. */
int eo_edge_probe(uint32_t count, const orc_splat* splats, const orc_settings* s, const float* pixel_xy, uint32_t* covered,
                  uint32_t* edge, float* s_xy);

#ifdef __cplusplus
}
#endif
#endif
