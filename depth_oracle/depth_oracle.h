/*
 * depth_oracle.h -- CPU ORACLE of bgs_render_depth_test (include/bgs.h: the splat depth d and the GreaterEqual test
 * against the scene's depth buffer).  TEST INFRASTRUCTURE ONLY: the product never links, loads or calls it.
 *
 * The walks are oracle/bgs_oracle.cpp's (this library compiles that file into itself and reuses its projection, sort,
 * binning and coverage decision), with the one addition of the depth test: a (pixel, splat) pair blends iff the
 * coverage decision holds and d >= scene[pixel].  `scene` is W x H floats, rows `pitch_bytes` apart; scene == NULL is
 * the walk without the test, bit for bit the oracle's.  FP policy as oracle/bgs_oracle.h.
 */
#ifndef DEPTH_ORACLE_H
#define DEPTH_ORACLE_H
#include <stdint.h>

#include "../oracle/bgs_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* d of gaussians ids[0 .. count): pz / pw of world_to_clip(model * pos) */
int dor_splat_depth(uint32_t n, const float* pos_vis, const orc_view* view, const orc_uniform* u, uint32_t count,
                    const uint32_t* ids, float* out);
/* ref_mode over a target (orc_render_ref_over), the test applied per fragment, back to front */
int dor_render_ref_over(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* scale_opacity,
                        const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* dst_init,
                        const float* scene, uint64_t pitch_bytes, float* out_rgba, int threads);
/* tile_mode frame (orc_render_tiles' image: over opaque black, alpha 1) */
int dor_render_tiles(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* scale_opacity,
                     const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* scene,
                     uint64_t pitch_bytes, float* out_rgba, int threads);
/* orc_blend_trace's per-pixel trace of the depth-tested walk */
int dor_blend_trace(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* scale_opacity,
                    const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* scene,
                    uint64_t pitch_bytes, orc_trace* out, int threads);
/* orc_coverage_probe with the test: pair j also needs splat_d[j] >= scene_d[j] to be covered (splat_d NULL: no test) */
int dor_coverage_probe(uint32_t count, const orc_splat* splats, const orc_settings* s, const float* pixel_xy,
                       const float* splat_d, const float* scene_d, orc_probe* out);

#ifdef __cplusplus
}
#endif
#endif
