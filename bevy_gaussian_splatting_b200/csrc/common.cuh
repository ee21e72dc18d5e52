// common.cuh -- shared device-side types and helpers of libbgs (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/bgs.h"

namespace bgs {

constexpr int TILE_PX = 16;           // 16x16-pixel raster tiles (a7)
constexpr float T_STOP = 1.0e-4f;     // a pixel stops once its transmittance drops below this

// Saturation bound of the entry and pair counts (n and n_pairs are < 2^30).
constexpr uint32_t LB_VMASK = (1u << 30) - 1u;

// Per-frame constants handed to the kernels by value (column-major matrices, as Bevy).
struct FrameConsts {
    float model[16];            // CloudUniform.transform
    float view_from_world[16];
    float clip_from_world[16];
    float cam[3];
    float W, H;                 // viewport.zw
    float p00, p11;             // clip_from_view[0].x, clip_from_view[1].y
    float global_opacity, global_scale;
    uint32_t color_space;
    uint32_t key_shift;         // 32 - radix_sort_depth_bits
    uint32_t gaussian_mode, rasterize_mode, aabb, adaptive, draw_mode;
    int Wi, Hi, tiles_x, tiles_y;
    uint32_t n_cloud;           // gaussians in the cloud
    uint32_t model_identity;    // CloudUniform.transform is exactly the identity (key-gen skips the multiply)
    float aabb_min[3], aabb_max[3];   // CloudUniform.min / .max (RasterizeMode::Position)
    uint32_t cov_pre;           // the cloud carries Covariance3dOpacityPacked128 records (f16.rs:131-170) instead of rotation + scale
    uint32_t aux;               // bgs_render_aux: the projection also emits the Depth and Normal colour sources
};

// The FrameConsts of one cloud (n_cloud gaussians, cov_pre its layout) under a uniform, a view and its settings: the one
// construction both the host (frame_consts, api.cu) and bgs_entity_list's expansion kernel (entity_list.cu) use, so a
// segment built on the device is bit for bit the one the host builds.  model_identity is a bitwise test, as memcmp
// is: -0.0 and NaN entries take the general path.
__host__ __device__ inline FrameConsts make_frame_consts(const bgs_view& view, const bgs_cloud_uniform& uni,
                                                         uint32_t radix_sort_depth_bits, uint32_t gaussian_mode,
                                                         uint32_t rasterize_mode, uint32_t aabb, uint32_t adaptive,
                                                         uint32_t draw_mode, uint32_t n_cloud, uint32_t cov_pre, uint32_t aux) {
    const int W = (int)view.viewport[2], H = (int)view.viewport[3];
    FrameConsts fc;
    memcpy(fc.model, uni.transform, 64);
    memcpy(fc.view_from_world, view.view_from_world, 64);
    memcpy(fc.clip_from_world, view.clip_from_world, 64);
    memcpy(fc.cam, view.world_position, 12);
    fc.W = view.viewport[2]; fc.H = view.viewport[3];
    fc.p00 = view.clip_from_view[0]; fc.p11 = view.clip_from_view[5];
    fc.global_opacity = uni.global_opacity; fc.global_scale = uni.global_scale;
    fc.color_space = uni.color_space;
    fc.key_shift = 32u - radix_sort_depth_bits;
    fc.gaussian_mode = gaussian_mode; fc.rasterize_mode = rasterize_mode; fc.aabb = aabb;
    fc.adaptive = adaptive; fc.draw_mode = draw_mode;
    fc.Wi = W; fc.Hi = H; fc.tiles_x = (W + TILE_PX - 1) / TILE_PX; fc.tiles_y = (H + TILE_PX - 1) / TILE_PX;
    fc.n_cloud = n_cloud;
    fc.aux = aux;
    fc.cov_pre = cov_pre;
    memcpy(fc.aabb_min, uni.aabb_min, 12); memcpy(fc.aabb_max, uni.aabb_max, 12);
    uint32_t identity = 1u;
    for (int i = 0; i < 16; ++i) {
        uint32_t bits;
        memcpy(&bits, &uni.transform[i], 4);
        if (bits != (i % 5 == 0 ? 0x3f800000u : 0u)) identity = 0u;
    }
    fc.model_identity = identity;
    return fc;
}

// A scene frame's segment table (bgs_render_scene, _scene_4d, _entities).  Segment j holds cloud j's gaussians at global
// indices [offset, offset + n); its FrameConsts carry the frame-wide values and entity j's settings, uniform and layout
// (n_cloud is the scene's N).  The scene
// kernels take it by value: 64 segments are ~22 KB of kernel parameters (CUDA >= 12.1 allows 32 KB on sm_90), so a
// queued frame's table lives in its own launches and no later frame can overwrite it.
struct SceneSeg {
    FrameConsts fc;
    const float4* pos;          // the cloud's position plane and blocks (cloud_layout.cuh)
    const void* blocks;
    uint32_t offset, n;
    uint32_t group;             // the projection launch the segment belongs to (api.cu: one per kernel instantiation)
};
struct SceneTable {
    uint32_t k;                 // segments, 1 .. BGS_SCENE_MAX_CLOUDS
    uint32_t n_total;           // N = sum of n
    SceneSeg seg[BGS_SCENE_MAX_CLOUDS];
    // the segment of global index g < N: the last j with offset <= g (empty segments share their successor's offset)
    __device__ __forceinline__ uint32_t find(uint32_t g) const {
        uint32_t lo = 0u, hi = k;
        while (hi - lo > 1u) {
            const uint32_t mid = (lo + hi) >> 1;
            if (seg[mid].offset <= g) lo = mid; else hi = mid;
        }
        return lo;
    }
    // find() for a g that only grows from one call to the next (j: the previous answer)
    __device__ __forceinline__ uint32_t advance(uint32_t j, uint32_t g) const {
        while (j + 1u < k && seg[j + 1u].offset <= g) ++j;
        return j;
    }
};

// bgs_render_entities_many's segment table, which lives in device memory (one copy per frame from the host) so that k is
// not bounded by the kernel-parameter limit: k segments seg[0 .. k) as SceneTable's, and beside them their offsets (what
// find and advance read: one word per step instead of a SceneSeg), times, num_classes and blend kinds.  Its kernels take
// this handle by value.
struct TemporalConsts;
struct SceneTableDev {
    uint32_t k;                 // segments, 1 .. BGS_ENTITIES_MANY_MAX
    uint32_t n_total;           // N = sum of n
    const SceneSeg* seg;
    const uint32_t* offset;     // seg[j].offset
    const TemporalConsts* times;
    const uint32_t* classes;    // num_classes of each segment
    const uint32_t* kinds;      // SegmentKinds::kind of each segment
    __device__ __forceinline__ uint32_t find(uint32_t g) const {
        uint32_t lo = 0u, hi = k;
        while (hi - lo > 1u) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(offset + mid) <= g) lo = mid; else hi = mid;
        }
        return lo;
    }
    __device__ __forceinline__ uint32_t advance(uint32_t j, uint32_t g) const {
        while (j + 1u < k && __ldg(offset + j + 1u) <= g) ++j;
        return j;
    }
};

// bgs_entity_list's compact record of one entity (device memory, 160 B): what its segment takes from the entity alone.
// entity_list.cu expands it with the frame's view into the segment; its offset, times, num_classes and kind live in the
// table's own arrays beside it.
struct EntityRec {
    bgs_cloud_uniform uni;      // transform column-major
    uint32_t gaussian_mode, rasterize_mode, aabb, adaptive, draw_mode;   // bgs_entity_settings'
    uint32_t n;                 // the cloud's gaussians
    uint32_t group;             // SceneSeg::group
    uint32_t cov_pre;           // FrameConsts::cov_pre
    const float4* pos;
    const void* blocks;
};
static_assert(sizeof(EntityRec) == 160, "EntityRec is 160 bytes");

// The projection group of Gaussian4d segments: project_group gives the 3D layouts 0 .. 7 (f16 bit, SH degree << 1), so
// 4D segments never fall into a 3D launch, and splat_depth_scene leaves their depths to the 4D projection, which takes
// them from the moved positions.
constexpr uint32_t PROJECT_GROUP_4D = 8u;
// a 3D group's bit for the Classification / OpticalFlow / Velocity colour kernel (groups 16 .. 23)
constexpr uint32_t ENTITY_MODES = 16u;

// bgs_render_extras as the Classification / OpticalFlow projection reads it: an argument of project_modes_kernel, the
// Gaussian4d kernels and the scene kernels, so project_kernel's arguments and code stay what they were.
struct ModeConsts {
    float prev_clip_from_world[16];   // the view's clip_from_world of the previous frame (column-major)
    float delta_time;                 // > 0, finite
    uint32_t num_classes;             // > 0
};

// bgs_render_4d's time, as the Gaussian4d projection (project_4d_kernel, an argument of its own) reads it
struct TemporalConsts {
    float time;          // bgs_cloud_uniform.time
    float time_future;   // time + 1e-3f: RasterizeMode::Velocity's second conditioning
    float duration;      // time_stop - time_start (finite, non-zero): the time terms' theta = dt / duration
};

// A scene's per-segment times (t[j] is segment j's; only 4D segments read theirs).  An argument of project_4d_scene_kernel
// alone (768 B beside the ~22 KB segment table).
struct SceneTimes {
    TemporalConsts t[BGS_SCENE_MAX_CLOUDS];
};

// A scene's per-segment num_classes (n[j] is segment j's).  An argument of the scene projection kernels, as SceneTimes
// is, so FrameConsts -- and the parameters of every single-cloud kernel -- stay as they are.
struct SceneClasses {
    uint32_t n[BGS_SCENE_MAX_CLOUDS];
};

// The blend kind of each segment of a mixed-geometry frame (bgs_render_entities): 0 = quad-uv (OBB), 1 = conic (3DGS / 4D
// with aabb), 2 = surfel (2DGS with aabb); raster.cu's class launch tags each compact slot with its segment's kind.
// Bit 2 of a kind (BOX_KIND) is the segment's bounding-box overlay, read only by the overlay's mixed blend.
constexpr uint32_t BOX_KIND = 4u;
struct SegmentKinds {
    uint32_t k;
    uint32_t offset[BGS_SCENE_MAX_CLOUDS];
    uint32_t kind[BGS_SCENE_MAX_CLOUDS];
};

// A views frame (bgs_render_views): v views of one entity list.  View i owns segments i k .. i k + k - 1 and the global
// indices [i n_view, (i + 1) n_view), and the global tile ids [tile0[i], tile0[i + 1]), row-major in its own
// tiles_x x tiles_y grid.  Binning reads the tile geometry; the blend also the view's size, target and depth buffer (scene
// NULL: no depth test), and on aux frames (bgs_render_views_aux) its depth and normal targets.  Taken by value
// (__grid_constant__, ~3.8 KB of kernel parameters) like the segment table.
constexpr uint32_t MAX_VIEWS = BGS_SCENE_MAX_CLOUDS;
struct ViewTable {
    uint32_t v;                 // views, 2 .. MAX_VIEWS (0: not a views frame)
    uint32_t n_view;            // global indices per view (the entity list's N)
    uint32_t tile0[MAX_VIEWS + 1];   // tile0[v] = every view's tiles
    int W[MAX_VIEWS], H[MAX_VIEWS], tiles_x[MAX_VIEWS], tiles_y[MAX_VIEWS];
    void* out[MAX_VIEWS];
    const float* scene[MAX_VIEWS];
    size_t pitch[MAX_VIEWS];
    void* out_depth[MAX_VIEWS];      // aux frames only
    void* out_normal[MAX_VIEWS];
    // the view of global index g < v n_view
    __device__ __forceinline__ uint32_t view_of(uint32_t g) const { return g / n_view; }
    // the view of global tile b < tile0[v]: the last i with tile0[i] <= b
    __device__ __forceinline__ uint32_t view_of_tile(uint32_t b) const {
        uint32_t lo = 0u, hi = v;
        while (hi - lo > 1u) {
            const uint32_t mid = (lo + hi) >> 1;
            if (tile0[mid] <= b) lo = mid; else hi = mid;
        }
        return lo;
    }
};
// sm_90 takes up to 32764 B of kernel parameters (CUDA >= 12.1): the kernels that take the view table (binning and the
// views blends) pass it with fewer than 256 B of other parameters
static_assert(sizeof(ViewTable) + 256 <= 32764, "a kernel taking the view table exceeds the sm_90 parameter limit");

// bgs_render_views_aux's Depth range of each view (depth_range_views_kernel), in the frame arena (cleared with it).
// View i's list is its visible entries in sort order, then its culled entries in ascending index; range[i] is
// (distance of its sorted[n - 1], distance of its sorted[1]), as FrameCounters' depth_min / depth_max are the
// single-view frame's.  The other fields are the pass's: positions p in the sorted payload are kept as ~p, so the
// cleared arena reads as "none yet" and a larger word is an earlier position.
struct ViewRanges {
    float2 range[MAX_VIEWS];
    unsigned long long first2[MAX_VIEWS];   // (~p0) << 32 | ~p1: the view's first two visible positions p0 < p1
    uint32_t last_p1[MAX_VIEWS];            // its last visible position + 1 (0: none)
    uint32_t n_vis[MAX_VIEWS];              // its visible entries
    uint32_t done;                          // CTAs past the pass (the last one computes the ranges)
};

// Projected splat record, 48 B, stored by front-to-back rank.
struct __align__(16) SplatRec {
    float cx, cy, ux, uy;       // centre (px), first row of the pixel-offset -> uv map
    float vx, vy;               // second row
    uint32_t bx, by;            // pixel bbox: lo | hi << 16 (inclusive); lo > hi = empty
    float r, g, b, op;          // linear rgb (unclamped), opacity * global_opacity
};
static_assert(sizeof(SplatRec) == 48, "SplatRec must be 48 bytes");

// Counters of one binning round.  A frame normally has ONE round (chunk 0 = all visible splats); frames whose
// splats cover many tiles each are binned / sorted / rasterised in several front-to-back rank chunks so that the
// rounds after every tile has saturated emit nothing (saturation-aware binning, see api.cu).
struct ChunkCounters {
    uint32_t n_pairs;           // (splat, tile) pairs emitted (clamped to capacity)
    uint32_t n_pairs_needed;    // pairs the round needs (may exceed capacity -> host regrows and redoes the frame)
    uint32_t barrier;           // grid barrier of bin_emit_coop (two uses per launch)
    uint32_t big_count;         // queue of large footprints (grows from the back of the queue arrays)
    uint32_t med_count;         // queue of medium footprints (grows from the front), drained 32 per warp
    uint32_t sort_barrier;      // grid barrier of the pair sort
    uint32_t skipped;           // 1 = the round emitted nothing because every tile had already saturated
    uint32_t pad[9];
};
static_assert(sizeof(ChunkCounters) == 64, "ChunkCounters is 64 bytes");
constexpr int MAX_CHUNKS = 5;         // rounds of a chunked frame (api.cu: CHUNK_FRAC)

// Device-resident per-frame counters (cleared at frame start).
struct FrameCounters {
    uint32_t n_sort;            // entries the depth sort runs over (n_vis, or N with SORT_ALL)
    uint32_t n_vis;             // in-frustum gaussians
    uint32_t tiles_done;        // tiles whose pixels have all saturated (chunked frames)
    uint32_t truncated;         // some round needed more pairs than the buffer holds: the blend leaves the target as it was
    uint32_t culled_min_inv;    // RasterizeMode::Depth: max over culled of (0xFFFFFFFF - index); 0 = none culled
    uint32_t culled_max_p1;     //                       max over culled of (index + 1);          0 = none culled
    float depth_min, depth_max; //                       distances of sorted[N-1] / sorted[1] (gaussian.wgsl:329-349)
    uint32_t barrier[2];        // grid barriers: [0] keygen_coop, [1] the depth sort
    ChunkCounters chunk[MAX_CHUNKS];
};

// flag/counter words exchanged between CTAs of one kernel: relaxed, GPU scope (L2 is the coherence point;
// ld/st.volatile would be SYSTEM scope)
__device__ __forceinline__ uint32_t ld_volatile(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// Grid-wide barrier for kernels launched with cudaLaunchCooperativeKernel (all CTAs co-resident).
// `bar` is zeroed by the per-frame clear; each use passes the cumulative arrival target.
__device__ __forceinline__ void grid_barrier(uint32_t* bar, uint32_t target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(bar, 1u);
        while (ld_volatile(bar) < target) { __nanosleep(32); }
        __threadfence();
    }
    __syncthreads();
}

// Sum of counts[0 .. upto) by the whole CTA (counts were published before a grid barrier).
template <int THREADS>
__device__ __forceinline__ uint32_t block_sum_prefix(const uint32_t* counts, uint32_t upto, uint32_t* s_red /*[THREADS/32]*/) {
    uint32_t v = 0u;
    for (uint32_t p = threadIdx.x; p < upto; p += THREADS) v += ld_volatile(counts + p);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t tot = 0u;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) tot += s_red[w];
    __syncthreads();
    return tot;
}

}  // namespace bgs
