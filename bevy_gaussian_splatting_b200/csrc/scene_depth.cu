// scene_depth.cu -- the splat depths of a depth-tested frame (bgs_render_depth_test, include/bgs.h).
//
// One thread per projection record: record r's depth d = world_to_clip(model * pos).z / .w lands at depths[r], indexed
// like the records (launch_project's index list and `by_slot` convention), so the blend kernels stage a splat's d from
// the same tile entry as its record.  A kernel of its own, enqueued only for depth-tested frames, so the projection
// kernels of every other frame stay as they are.  Compiled -fmad=false (project_math.cuh): d is bit-exact vs the oracle.
#include "project_math.cuh"
#include "entry_src.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int SD_THREADS = 256, SD_CTAS_PER_SM = 8;

template <class Src>
__device__ __forceinline__ void splat_depth_body(const Src& src, const FrameCounters* __restrict__ ctr,
                                                 float* __restrict__ depths) {
    const uint32_t n_vis = ctr->n_vis;
    for (uint32_t r = blockIdx.x * SD_THREADS + threadIdx.x; r < n_vis; r += gridDim.x * SD_THREADS) {
        const uint32_t id = src.entry(r, n_vis), j = src.seg(id);
        if (Src::SEGMENTED && !src.mine(j)) continue;
        const FrameConsts& fc = src.fc(j);
        const float4 p = __ldg(src.pos_at(j, id));
        float pw[4];
        mat4_point(fc.model, p.x, p.y, p.z, pw);   // the projection's full multiply (a -0 stays -0)
        depths[r] = splat_depth(fc, pw);
    }
}

__global__ void __launch_bounds__(SD_THREADS)
splat_depth_kernel(const float4* __restrict__ pos, const uint32_t* __restrict__ index_list, int by_slot,
                   const FrameCounters* __restrict__ ctr, FrameConsts fc, float* __restrict__ depths) {
    splat_depth_body(OneCloud{pos, fc, nullptr, index_list, by_slot}, ctr, depths);
}

// Scene frames: record r is compact slot r.  Every 3D group is this launch's, with either colour kernel (groups 0 .. 7
// and 16 .. 23, ENTITY_MODES); Gaussian4d segments are not: their projection writes their depths from the moved positions.
__global__ void __launch_bounds__(SD_THREADS)
splat_depth_scene_kernel(SceneTable tab, const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                         float* __restrict__ depths) {
    constexpr uint32_t groups_3d = ((1u << PROJECT_GROUP_4D) - 1u) * (1u | 1u << ENTITY_MODES);   // 0x00FF00FF
    splat_depth_body(SceneSrc{tab, groups_3d, slot_ids}, ctr, depths);
}

// bgs_render_entities_many: the same over a segment table in device memory
__global__ void __launch_bounds__(SD_THREADS)
splat_depth_many_kernel(SceneTableDev tab, const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                        float* __restrict__ depths) {
    constexpr uint32_t groups_3d = ((1u << PROJECT_GROUP_4D) - 1u) * (1u | 1u << ENTITY_MODES);
    splat_depth_body(SceneSrcDev{tab, groups_3d, slot_ids}, ctr, depths);
}

void launch_splat_depth(const float4* pos, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                        const FrameConsts& fc, float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream) {
    const uint32_t grid = persistent_grid(n_hint, SD_THREADS, SD_CTAS_PER_SM, sm_count);
    splat_depth_kernel<<<grid, SD_THREADS, 0, stream>>>(pos, index_list, by_slot, ctr, fc, depths);
}

void launch_splat_depth_scene(const SceneTable& tab, const uint32_t* slot_ids, const FrameCounters* ctr, float* depths,
                              uint32_t n_hint, int sm_count, cudaStream_t stream) {
    const uint32_t grid = persistent_grid(n_hint, SD_THREADS, SD_CTAS_PER_SM, sm_count);
    splat_depth_scene_kernel<<<grid, SD_THREADS, 0, stream>>>(tab, slot_ids, ctr, depths);
}

void launch_splat_depth_many(const SceneTableDev& tab, const uint32_t* slot_ids, const FrameCounters* ctr, float* depths,
                             uint32_t n_hint, int sm_count, cudaStream_t stream) {
    const uint32_t grid = persistent_grid(n_hint, SD_THREADS, SD_CTAS_PER_SM, sm_count);
    splat_depth_many_kernel<<<grid, SD_THREADS, 0, stream>>>(tab, slot_ids, ctr, depths);
}

}  // namespace bgs
