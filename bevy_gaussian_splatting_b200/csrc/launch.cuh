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
// bgs_render_entities_many's: the same over a segment table in device memory (fc: the frame-wide values)
int keygen_many_blocks_per_sm();
cudaError_t launch_keygen_many(const SceneTableDev& tab, const FrameConsts& fc, uint32_t* masks, uint32_t* keys_out,
                               uint32_t* ids_out, uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr, uint32_t* hist,
                               int hist_passes, uint32_t grid, cudaStream_t stream);
void launch_culled_flags_many(const SceneTableDev& tab, uint32_t* flags, cudaStream_t stream);
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
// scene frames (bgs_render_scene, _scene_4d, _entities): the projection group of a cloud's segments, and the depth range
uint32_t project_group(CloudLayout layout, uint32_t sh_degree);
void launch_depth_range_scene(const SceneTable& tab, const uint32_t* sorted_payload, const uint32_t* slot_ids, FrameCounters* ctr,
                              cudaStream_t stream);
// Gaussian4d clouds (bgs_render_4d): records as launch_project's, and the splat depths of depth-tested frames (depths
// non-null) from the moved positions
void launch_project_4d(const void* blocks, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                       const FrameConsts& fc, const ModeConsts& mc, const TemporalConsts& tc, SplatRec* recs, float* depths,
                       uint32_t n_hint, int sm_count, cudaStream_t stream);
// scene frames: the projection of the segments of one group (project_group, | ENTITY_MODES for the Classification /
// OpticalFlow / Velocity kernel; one launch), each with its own settings and num_classes; need_sh: some segment of the
// group reads the SH coefficients.  And the Gaussian4d segments' (PROJECT_GROUP_4D), each at its own times, with their
// splat depths from the moved positions (depths non-null).  view_ranges non-null (bgs_render_views_aux, k segments per
// view): each segment's Depth colours over its view's range.
void launch_project_scene(const SceneTable& tab, uint32_t group, bool need_sh, const SceneClasses& classes,
                          const ModeConsts& mc, const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs,
                          float4* extra, uint32_t n_hint, int sm_count, const float* cutoff_tab,
                          float4* aux /* bgs_render_entities_aux: each segment's depth / normal colours; else null */,
                          cudaStream_t stream, const ViewRanges* view_ranges = nullptr, uint32_t k = 0);
// bgs_render_views_aux: the Depth range of each of v views of n_view global indices (ViewRanges::range; the arena clear
// resets the rest), in place of launch_depth_range_scene
void launch_depth_range_views(const SceneTable& tab, uint32_t v, uint32_t n_view, const uint32_t* sorted_payload,
                              const uint32_t* slot_ids, const FrameCounters* ctr, ViewRanges* view_ranges, uint32_t n_hint,
                              int sm_count, cudaStream_t stream);
void launch_project_4d_scene(const SceneTable& tab, const SceneTimes& times, const SceneClasses& classes,
                             const ModeConsts& mc, const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs,
                             float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream);
// bgs_render_entities_many: the same over a segment table in device memory (its times and num_classes beside it); one
// launch_project_many per group, the 4D group included (depths: its splat depths)
void launch_depth_range_many(const SceneTableDev& tab, const uint32_t* sorted_payload, const uint32_t* slot_ids,
                             FrameCounters* ctr, cudaStream_t stream);
void launch_project_many(const SceneTableDev& tab, uint32_t group, bool need_sh, const ModeConsts& mc,
                         const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs, float4* extra,
                         float* depths, uint32_t n_hint, int sm_count, const float* cutoff_tab, cudaStream_t stream);
// bin.cu
int bin_coop_blocks_per_sm();
cudaError_t launch_bin_emit_coop(const SplatRec* recs, const uint32_t* perm, FrameCounters* ctr, ChunkCounters* cc,
                                 uint32_t frac_a, uint32_t frac_b, uint32_t num_tiles_total, uint32_t* block_cnt,
                                 int tiles_x, uint32_t capacity, uint32_t* pair_keys, uint32_t* pair_vals,
                                 uint32_t* q_rank, uint32_t* q_off, uint32_t q_cap, uint32_t grid,
                                 uint32_t* sticky_need, cudaStream_t stream);
// bgs_render_views: one round, each splat into its view's tiles (slot_ids: compact slot -> global index)
cudaError_t launch_bin_emit_views(const SplatRec* recs, const uint32_t* perm, FrameCounters* ctr, ChunkCounters* cc,
                                  uint32_t num_tiles_total, uint32_t* block_cnt, uint32_t capacity, uint32_t* pair_keys,
                                  uint32_t* pair_vals, uint32_t* q_rank, uint32_t* q_off, uint32_t q_cap, uint32_t grid,
                                  uint32_t* sticky_need, const uint32_t* slot_ids, const ViewTable& vt, int sm_count,
                                  cudaStream_t stream);
// scene_depth.cu
void launch_splat_depth(const float4* pos, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                        const FrameConsts& fc, float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream);
void launch_splat_depth_scene(const SceneTable& tab, const uint32_t* slot_ids, const FrameCounters* ctr, float* depths,
                              uint32_t n_hint, int sm_count, cudaStream_t stream);
void launch_splat_depth_many(const SceneTableDev& tab, const uint32_t* slot_ids, const FrameCounters* ctr, float* depths,
                             uint32_t n_hint, int sm_count, cudaStream_t stream);
// raster.cu.  A one-round frame's blend of the sorted pairs `tile_entries` (per tile: `ranges`) into `out`, W x H in
// tiles_x x tiles_y tiles, in `format` (BGS_FORMAT_* | output mode << 8).  mode 0..2: one blend kind for every splat;
// 3 / 4 (bgs_render_entities): mixed kinds, read from `kinds` (one byte per record), 4 when some splat is a surfel.  box:
// the bounding-box overlay (BGS_FLAG_VISUALIZE_BOUNDING_BOX) on every splat, or on a mixed frame on those whose kinds byte
// has bit 2 set.  large_footprints: the quad-uv blend of a plain single-view frame takes raster2_kernel.  aux non-null
// (bgs_render_aux, _entities_aux, _views_aux): also the depth and normal frames, into out_depth / out_normal.  scene
// non-null (bgs_scene_depth): the depth test of the splat depths splat_d (indexed like the records) against that buffer.
// views non-null (bgs_render_views, _views_aux): one CTA per global tile of every view (views->tile0[views->v]), each into
// its view's targets and depth buffer (scene is then view 0's).  pick non-null (bgs_render_entities_pick): also, per pixel,
// the pick record (include/bgs.h's bgs_pick) into pick->out, from the record's global index (slot_ids) and segment (seg:
// offsets and k) and its depth splat_d[record] (written with or without a depth buffer).
struct PickArgs {
    uint4* out;
    const uint32_t* slot_ids;
    SegmentKinds seg;
    // global index g as (segment, index within it): the last j with offset <= g (SceneTable::find)
    __device__ __forceinline__ uint2 locate(uint32_t g) const {
        uint32_t lo = 0u, hi = seg.k;
        while (hi - lo > 1u) {
            const uint32_t mid = (lo + hi) >> 1;
            if (seg.offset[mid] <= g) lo = mid; else hi = mid;
        }
        return make_uint2(lo, g - seg.offset[lo]);
    }
};
// bgs_render_entities_many's pick frame: the segments are the device table's
struct PickArgsDev {
    uint4* out;
    const uint32_t* slot_ids;
    SceneTableDev tab;
    __device__ __forceinline__ uint2 locate(uint32_t g) const {
        const uint32_t j = tab.find(g);
        return make_uint2(j, g - __ldg(tab.offset + j));
    }
};
static_assert(sizeof(bgs_pick) == sizeof(uint4), "a pick record is stored as one uint4");
struct BlendArgs {
    int mode = 0;
    bool box = false;
    bool large_footprints = false;
    const SplatRec* recs = nullptr;
    const float4* extra = nullptr;
    const uint32_t* tile_entries = nullptr;
    const uint2* ranges = nullptr;
    int W = 0, H = 0, tiles_x = 0, tiles_y = 0;
    void* out = nullptr;
    uint32_t format = 0;
    const float4* aux = nullptr;
    void* out_depth = nullptr;
    void* out_normal = nullptr;
    const uint32_t* truncated = nullptr;
    const float* splat_d = nullptr;
    const float* scene = nullptr;
    size_t pitch = 0;
    const unsigned char* kinds = nullptr;
    const ViewTable* views = nullptr;
    bool raw = false;   // (bgs_render_shutter, with views: each view's pixels' raw (C, T) as float4 into its out, no format)
    const PickArgs* pick = nullptr;
    const PickArgsDev* pick_dev = nullptr;   // (bgs_render_entities_pick_many: in place of pick)
};
void launch_raster(const BlendArgs& a, cudaStream_t stream);
// one front-to-back round of a chunked frame (a's single-view quad-uv blend, depth test included): each pixel's blend state
// in `state` between rounds, tile_done / tiles_done the tiles saturated so far
void launch_raster_round(const BlendArgs& a, float4* state, unsigned char* tile_done, uint32_t* tiles_done, int first, int last,
                         cudaStream_t stream);
// a mixed-geometry frame's blend kind of each compact slot (records n_vis of ctr), from its segment's
void launch_segment_kinds(const SegmentKinds& kinds, const uint32_t* slot_ids, const FrameCounters* ctr, unsigned char* out,
                          uint32_t n_hint, int sm_count, cudaStream_t stream);
void launch_segment_kinds_many(const SceneTableDev& tab, const uint32_t* slot_ids, const FrameCounters* ctr, unsigned char* out,
                               uint32_t n_hint, int sm_count, cudaStream_t stream);
// shutter.cu: bgs_render_shutter's resolve.  sub: s sub-frames of wh pixels each, pixel p of sub-frame i at sub[i wh + p],
// its raw (C, T) as the blend stored it; out: the frame, in `format` (raster.cu's: BGS_FORMAT_* | output mode << 8), pixel p
// the pixel write of the pairwise mean (include/bgs.h).  Writes nothing when *truncated is set (the frame is rendered again).
// s in 2 .. MAX_VIEWS.
void launch_shutter_resolve(const float4* sub, uint32_t s, uint32_t wh, void* out, uint32_t format, const uint32_t* truncated,
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
// view_select.cu: bgs_cloud_select_in_view's pass (fc: the frame constants of the cloud, uniform and view; mask Hi x Wi
// bytes on the device; mode as the mesh selection's; *inside += the gaussians inside)
void launch_view_select(CloudView cloud, uint32_t n, const FrameConsts& fc, const uint8_t* mask, uint32_t mode,
                        uint32_t* inside, cudaStream_t stream);
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
// transform.cu: bgs_cloud_transform's constants (cloud.cu: transform_params; the rule: include/bgs.h) -- the column-major
// matrix, q_R (w, x, y, z), s, and E_l = D_l^T row-major for the SH bands 1..3 -- and its pass; bgs_cloud_bounds' pass
// (words: min keys x, y, z, preset to 0xFFFFFFFF | max keys x, y, z, preset to 0 | count, preset to 0; a key is the f32's
// bits with the sign bit flipped when clear and every bit flipped when set)
struct TransformParams {
    float m[16];
    float q[4];
    float s;
    float sh1[9], sh2[25], sh3[49];
};
void launch_transform(CloudLayout layout, uint32_t sh_degree, CloudView cloud, uint32_t n, const TransformParams& p,
                      uint32_t selected_only, cudaStream_t stream);
void launch_bounds(const float4* pos, uint32_t n, uint32_t selected_only, uint32_t* words, int sm_count, cudaStream_t stream);
// interpolate.cu
void launch_interpolate(CloudLayout layout, uint32_t sh_degree, CloudView lhs, CloudView rhs, uint32_t n, float t, CloudView out, cudaStream_t stream);
// khr.cu: glTF component codes, the decode's rule bits (words[0]; words[1] counts zero-length quaternions), one accessor
// as the kernel reads it (its span's device copy), and a primitive's accessors (bands: SH coefficients per channel, 0
// for none; sh_units: 16 B units of the staged SH plane per gaussian)
enum : uint32_t { KHR_I8 = 5120, KHR_U8 = 5121, KHR_I16 = 5122, KHR_U16 = 5123, KHR_F32 = 5126 };
enum : uint32_t { KHR_BAD_POSITION = 1, KHR_BAD_ROTATION = 2, KHR_BAD_SCALE = 4, KHR_BAD_OPACITY = 8, KHR_BAD_SH = 16, KHR_BAD_COLOR = 32 };
struct KhrSrc {
    const uint8_t* data;
    uint32_t stride, type, normalized;
};
struct KhrDecode {
    KhrSrc position, rotation, scale, opacity, color, sh[16];
    uint32_t n, bands, sh_units;
};
// the staged planes of an f32 (so non-null) or f16 (rot: the packed second record) cloud
void launch_khr_decode(const KhrDecode& k, bool f16, float4* pos, void* sh, void* rot, void* so, uint32_t* words, cudaStream_t stream);
// entity_list.cu: bgs_entity_list's expansion of k records into segments (one launch per frame), and its edits' scatter
// of records (count entities, at the distinct indices idx) and of row-major transforms into records dst[0 .. count)
struct EntityListUpload {
    const uint32_t* idx;
    const EntityRec* recs;
    const uint32_t* offset;
    const TemporalConsts* times;
    const uint32_t* classes;
    const uint32_t* kinds;      // SegmentKinds::kind without the frame's overlay flag
};
struct EntityListArrays {
    EntityRec* recs;
    uint32_t* offset;
    TemporalConsts* times;
    uint32_t* classes;
    uint32_t* kinds;            // ... and kinds_box with BOX_KIND set on every entity (frames with the frame-wide overlay)
    uint32_t* kinds_box;
};
cudaError_t launch_entity_list_expand(const EntityRec* recs, const uint32_t* offset, uint32_t k, const bgs_view& view,
                                      uint32_t radix_sort_depth_bits, uint32_t n_total, SceneSeg* seg, cudaStream_t stream);
cudaError_t launch_entity_list_scatter(const EntityListUpload& u, uint32_t count, const EntityListArrays& a, cudaStream_t stream);
cudaError_t launch_entity_list_transforms(const float* m, uint32_t count, EntityRec* dst, cudaStream_t stream);
}  // namespace bgs
