// scene_depth.cu -- the splat depths of a depth-tested frame (bgs_render_depth_test, include/bgs.h).
//
// One thread per projection record: record r's depth d = world_to_clip(model * pos).z / .w lands at depths[r], indexed
// like the records (launch_project's index list and `by_slot` convention), so the blend kernels stage a splat's d from
// the same tile entry as its record.  A kernel of its own, enqueued only for depth-tested frames, so the projection
// kernels of every other frame stay as they are.  Compiled -fmad=false (project_math.cuh): d is bit-exact vs the oracle.
#include "project_math.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int SD_THREADS = 256;

__global__ void __launch_bounds__(SD_THREADS)
splat_depth_kernel(const float4* __restrict__ pos, const uint32_t* __restrict__ index_list, int by_slot,
                   const FrameCounters* __restrict__ ctr, FrameConsts fc, float* __restrict__ depths) {
    const uint32_t n_vis = ctr->n_vis;
    for (uint32_t r = blockIdx.x * SD_THREADS + threadIdx.x; r < n_vis; r += gridDim.x * SD_THREADS) {
        const uint32_t id = by_slot ? __ldg(index_list + r) : __ldg(index_list + (n_vis - 1u - r));
        const float4 p = __ldg(pos + id);
        float pw[4];
        mat4_point(fc.model, p.x, p.y, p.z, pw);   // the projection's full multiply (a -0 stays -0)
        depths[r] = splat_depth(fc, pw);
    }
}

// bgs_render_scene: record r is compact slot r, its global index in segment j (common.cuh).  Gaussian4d segments
// (bgs_render_scene_4d) are skipped: their projection writes their depths from the moved positions.
__global__ void __launch_bounds__(SD_THREADS)
splat_depth_scene_kernel(SceneTable tab, const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                         float* __restrict__ depths) {
    const uint32_t n_vis = ctr->n_vis;
    for (uint32_t r = blockIdx.x * SD_THREADS + threadIdx.x; r < n_vis; r += gridDim.x * SD_THREADS) {
        const uint32_t g = __ldg(slot_ids + r);
        const SceneSeg& s = tab.seg[tab.find(g)];
        if (s.group == PROJECT_GROUP_4D) continue;
        const float4 p = __ldg(s.pos + (g - s.offset));
        float pw[4];
        mat4_point(s.fc.model, p.x, p.y, p.z, pw);
        depths[r] = splat_depth(s.fc, pw);
    }
}

void launch_splat_depth(const float4* pos, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                        const FrameConsts& fc, float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream) {
    // grid-stride over the visible count, which only the device knows: sized by the hint, at most 8 CTAs per SM
    uint32_t grid = (n_hint + SD_THREADS - 1) / SD_THREADS;
    if (grid > (uint32_t)(8 * sm_count)) grid = (uint32_t)(8 * sm_count);
    if (grid < 1u) grid = 1u;
    splat_depth_kernel<<<grid, SD_THREADS, 0, stream>>>(pos, index_list, by_slot, ctr, fc, depths);
}

void launch_splat_depth_scene(const SceneTable& tab, const uint32_t* slot_ids, const FrameCounters* ctr, float* depths,
                              uint32_t n_hint, int sm_count, cudaStream_t stream) {
    uint32_t grid = (n_hint + SD_THREADS - 1) / SD_THREADS;
    if (grid > (uint32_t)(8 * sm_count)) grid = (uint32_t)(8 * sm_count);
    if (grid < 1u) grid = 1u;
    splat_depth_scene_kernel<<<grid, SD_THREADS, 0, stream>>>(tab, slot_ids, ctr, depths);
}

}  // namespace bgs
