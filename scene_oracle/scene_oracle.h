/*
 * scene_oracle.h -- CPU ORACLE of bgs_render_scene (include/bgs.h).  TEST INFRASTRUCTURE ONLY: only tests/ and
 * scripts/ may load it.
 *
 * The joint rule restated over the oracle's per-gaussian functions (oracle/bgs_oracle.h, same FP policy): cloud j's
 * gaussians take global indices o_j + i; each is keyed and projected by the oracle with its own cloud's planes and
 * uniform; the depth sort is stable over (key, global index) across all clouds; Depth colouring takes its range from
 * sorted[1] / sorted[N-1] of that joint list; binning and the blend (tile_mode), or the reference's back-to-front pass
 * (ref_mode), then run on the joint record set exactly as orc_render_tiles / orc_render_ref_over do for one cloud.
 */
#ifndef SCENE_ORACLE_H
#define SCENE_ORACLE_H
#include "../oracle/bgs_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* One listed cloud: its planes as the oracle reads them (sh: 48 floats per gaussian, zero-padded below degree 3; f16
 * clouds decoded), its uniform, and whether its planes hold decoded covariance records (orc_settings.reserved bit 0 for
 * this cloud alone). */
typedef struct {
    uint32_t n;
    uint32_t cov_pre;
    const float* pos_vis;
    const float* sh;
    const float* rot;
    const float* scale_opacity;
    orc_uniform u;
} sor_cloud;

/* N * 2 words (key, global index): the joint sorted entry list, culled entries last in ascending global index. */
int sor_sorted_entries(uint32_t k, const sor_cloud* clouds, const orc_view* view, uint32_t depth_bits, uint32_t* out);

/* orc_render_tiles over the joint record set (out_rgba may be NULL); records (n_vis, optional) in front-to-back rank. */
int sor_render_tiles(uint32_t k, const sor_cloud* clouds, const orc_view* view, const orc_settings* s, float* out_rgba,
                     uint32_t* tile_ranges, uint32_t* tile_entries, uint64_t cap, uint64_t* n_pairs, uint32_t* n_vis,
                     uint32_t* rank_to_id, orc_splat* records, int threads);

/* orc_render_ref_over over the joint record set: back to front, no tiles, no early-out, over dst_init (NULL: opaque
 * black). */
int sor_render_ref_over(uint32_t k, const sor_cloud* clouds, const orc_view* view, const orc_settings* s,
                        const float* dst_init, float* out_rgba, int threads);

#ifdef __cplusplus
}
#endif
#endif
