// launch.cuh -- the host entry points of libbgs's kernels: one declaration each, included by the .cu file that defines
// it and by the host code that calls it (api.cu, cloud.cu), so a signature that drifts fails to compile.
#pragma once
#include "cloud_layout.cuh"

namespace bgs {
// keygen.cu
void launch_keygen_all(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* keys_out, uint32_t* ids_out,
                       FrameCounters* ctr, cudaStream_t stream);
int keygen_coop_blocks_per_sm();
cudaError_t launch_keygen_coop(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* masks, uint32_t* keys_out,
                               uint32_t* ids_out, uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr,
                               uint32_t* hist, int hist_passes, uint32_t grid, cudaStream_t stream);
void launch_culled_flags(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* flags, cudaStream_t stream);
// bgs_render_scene's key-gen (one cooperative launch over the segment table's N global indices) and debug flags
int keygen_scene_blocks_per_sm();
cudaError_t launch_keygen_scene(const SceneTable& tab, uint32_t* masks, uint32_t* keys_out, uint32_t* ids_out,
                                uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr, uint32_t* hist, int hist_passes,
                                uint32_t grid, cudaStream_t stream);
void launch_culled_flags_scene(const SceneTable& tab, uint32_t* flags, cudaStream_t stream);
// radix.cu
uint32_t radix_num_tiles(uint32_t capacity);
int radix_coop_blocks_per_sm(int items);
cudaError_t launch_radix_sort(uint32_t* keys0, uint32_t* vals0, uint32_t* keys1, uint32_t* vals1, const uint32_t* n_ptr,
                              uint32_t capacity, uint32_t n_hint, uint32_t* hist, int compute_hist, void* status,
                              size_t status_stride, uint32_t epoch, uint32_t* barrier, int passes, int shift0, uint2* ranges,
                              int sm_count, int coop_per_sm, cudaStream_t stream);
// project.cu
void launch_depth_range(const float4* pos, uint32_t n, const uint32_t* sorted_payload, const uint32_t* slot_ids,
                        FrameCounters* ctr, const FrameConsts& fc, cudaStream_t stream);
void launch_repack(CloudLayout layout, uint32_t sh_degree, const void* sh /* staged: staged_bytes per gaussian */, const void* rot, const void* so, const void* tt /* 4D only */,
                   uint32_t n, CloudView cloud, cudaStream_t stream);
void launch_project(CloudLayout layout, uint32_t sh_degree, const void* blocks, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                    const FrameConsts& fc, SplatRec* recs, float4* extra, uint32_t n_hint, int sm_count,
                    const float* cutoff_tab, float4* aux, const ModeConsts* modes /* null: project_kernel */,
                    cudaStream_t stream);
void launch_cutoff_table(float* tab, cudaStream_t stream);
// bgs_render_scene: the projection of the segments whose project_group is `group` (one launch), and the depth range
uint32_t project_group(CloudLayout layout, uint32_t sh_degree);
void launch_project_scene(const SceneTable& tab, uint32_t group, const uint32_t* slot_ids, const FrameCounters* ctr,
                          SplatRec* recs, float4* extra, uint32_t n_hint, int sm_count, const float* cutoff_tab,
                          const ModeConsts* modes /* null: project_scene_kernel */, cudaStream_t stream);
void launch_depth_range_scene(const SceneTable& tab, const uint32_t* sorted_payload, const uint32_t* slot_ids, FrameCounters* ctr,
                              cudaStream_t stream);
// Gaussian4d clouds (bgs_render_4d): records as launch_project's, and the splat depths of depth-tested frames (depths
// non-null) from the moved positions
void launch_project_4d(const void* blocks, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                       const FrameConsts& fc, const ModeConsts& mc, const TemporalConsts& tc, SplatRec* recs, float* depths,
                       uint32_t n_hint, int sm_count, cudaStream_t stream);
// bgs_render_scene_4d: the projection of every segment in PROJECT_GROUP_4D (one launch), each at its own times, and their
// splat depths from the moved positions (depths non-null)
void launch_project_4d_scene(const SceneTable& tab, const SceneTimes& times, const uint32_t* slot_ids, const FrameCounters* ctr,
                             const ModeConsts& mc, SplatRec* recs, float* depths, uint32_t n_hint, int sm_count,
                             cudaStream_t stream);
// bgs_render_entities frames whose entities disagree: the projection of the segments of one group (project_group, |
// ENTITY_MODES for the Classification / OpticalFlow / Velocity kernel), each with its own settings and num_classes;
// need_sh: some segment of the group reads the SH coefficients.  And the 4D segments' (PROJECT_GROUP_4D).
void launch_project_entities(const SceneTable& tab, uint32_t group, bool need_sh, const SceneClasses& classes,
                             const ModeConsts& mc, const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs,
                             float4* extra, uint32_t n_hint, int sm_count, const float* cutoff_tab, cudaStream_t stream);
void launch_project_4d_entities(const SceneTable& tab, const SceneTimes& times, const SceneClasses& classes,
                                const ModeConsts& mc, const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs,
                                float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream);
// bin.cu
int bin_coop_blocks_per_sm();
cudaError_t launch_bin_emit_coop(const SplatRec* recs, const uint32_t* perm, FrameCounters* ctr, ChunkCounters* cc,
                                 uint32_t frac_a, uint32_t frac_b, uint32_t num_tiles_total, uint32_t* block_cnt,
                                 int tiles_x, uint32_t capacity, uint32_t* pair_keys, uint32_t* pair_vals,
                                 uint32_t* q_rank, uint32_t* q_off, uint32_t q_cap, uint32_t grid,
                                 uint32_t* sticky_need, cudaStream_t stream);
// scene_depth.cu
void launch_splat_depth(const float4* pos, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                        const FrameConsts& fc, float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream);
void launch_splat_depth_scene(const SceneTable& tab, const uint32_t* slot_ids, const FrameCounters* ctr, float* depths,
                              uint32_t n_hint, int sm_count, cudaStream_t stream);
// raster.cu.  ZTestArgs: a depth-tested frame's splat depths (indexed like the records) and the scene's depth buffer
// (bgs_scene_depth); scene == nullptr blends without the test.
struct ZTestArgs {
    const float* splat_d = nullptr;
    const float* scene = nullptr;
    size_t pitch = 0;
};
// mode 0..2: one blend kind for every splat; 3 / 4 (bgs_render_entities): mixed kinds, read from `kinds` (one byte per
// record), 4 when some splat is a surfel
void launch_raster(int mode, bool large_footprints, const SplatRec* recs, const float4* extra, const uint32_t* tile_entries,
                   const uint2* ranges, int W, int H, int tiles_x, int tiles_y, void* out, uint32_t format,
                   const float4* aux, void* out_depth, void* out_normal, const uint32_t* truncated, const ZTestArgs& zt,
                   cudaStream_t stream, const unsigned char* kinds = nullptr);
// a mixed-geometry frame's blend kind of each compact slot (records n_vis of ctr), from its segment's
void launch_segment_kinds(const SegmentKinds& kinds, const uint32_t* slot_ids, const FrameCounters* ctr, unsigned char* out,
                          uint32_t n_hint, int sm_count, cudaStream_t stream);
void launch_raster_round(const SplatRec* recs, const uint32_t* tile_entries, const uint2* ranges, int W, int H, int tiles_x,
                         int tiles_y, void* out, uint32_t format, float4* state, unsigned char* tile_done,
                         uint32_t* tiles_done, const uint32_t* truncated, int first, int last, const ZTestArgs& zt,
                         cudaStream_t stream);
// select.cu
uint32_t select_num_buckets(uint32_t n);
int select_sort_passes(uint32_t n_buckets);
void launch_select_keys(const float4* pos, uint32_t n, float radius, uint32_t n_buckets, uint32_t* keys, uint32_t* vals,
                        uint32_t* n_sort, cudaStream_t stream);
void launch_select_count(CloudView cloud, const uint32_t* ids, const uint2* ranges, uint32_t n, float radius, uint32_t n_buckets,
                         float r2, uint32_t threshold, float4* spos, uint32_t* selected, cudaStream_t stream);
void launch_select_fill(CloudView cloud, uint32_t n, float v, cudaStream_t stream);
// mesh_select.cu
size_t mesh_words_bytes();
size_t mesh_rec_bytes();
void launch_mesh_setup(const float* verts, const uint32_t* idx, uint32_t nt, void* bin_rec, void* bin_box, void* glob_rec, void* words,
                       cudaStream_t stream);
void launch_mesh_levels(const void* bin_box, const void* words_host, void* words, cudaStream_t stream);
void mesh_pick_level(const void* words_host, int* level, uint64_t* pairs, uint32_t* cells);
void launch_mesh_emit(const void* bin_box, const void* words_host, int level, uint32_t* keys, uint32_t* vals, void* words,
                      cudaStream_t stream);
uint32_t* mesh_words_pairs(void* words);
uint32_t* mesh_words_barrier(void* words);
uint32_t* mesh_words_inside(void* words);
uint32_t mesh_words_n_bin(const void* words_host);
void launch_mesh_count(CloudView cloud, uint32_t n, const float* mesh_from_cloud, const void* bin_rec, const void* glob_rec,
                       const uint32_t* cell_tri, const uint2* ranges, const void* words_host, int level, uint32_t mode, void* words,
                       cudaStream_t stream);
// particles.cu
void launch_particle_step(void* behaviors, uint32_t count, float dt, CloudView cloud, cudaStream_t stream);
// subset.cu
uint32_t subset_num_ctas(uint32_t n);
void launch_subset_count(const float4* pos, uint32_t n, uint32_t* mask, uint32_t* cta_cnt, uint32_t* total, cudaStream_t stream);
void launch_subset_scatter(CloudLayout layout, uint32_t sh_degree, CloudView src, uint32_t n, const uint32_t* mask, const uint32_t* cta_off,
                           CloudView dst, cudaStream_t stream);
void launch_subset_gather(CloudLayout layout, uint32_t sh_degree, CloudView src, const uint32_t* idx, uint32_t k, CloudView dst, cudaStream_t stream);
void launch_unpack(CloudLayout layout, uint32_t sh_degree, CloudView cloud, uint32_t lo, uint32_t m, void* sh, void* rot, void* so,
                   void* tt /* 4D only */, cudaStream_t stream);
// interpolate.cu
void launch_interpolate(CloudLayout layout, uint32_t sh_degree, CloudView lhs, CloudView rhs, uint32_t n, float t, CloudView out, cudaStream_t stream);
}  // namespace bgs
