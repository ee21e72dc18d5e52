// view_select.cu -- bgs_cloud_select_in_view (include/bgs.h): selection through a screen-space mask.
//
// One thread per gaussian, one streaming pass over the position plane: the projection's centre of the gaussian with this
// uniform and view (the full model multiply, in_frustum, then cx = ndc.x hw + hw, cy = hh - ndc.y hh, exactly as
// project_one computes the record), and the mask byte under it.  Compiled -fmad=false (project_math.cuh), so the
// frustum decision and (cx, cy) are bit for bit the projection's.
#include "project_math.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int VS_THREADS = 256;

// mode 0 (replace): lane = inside ? 1 : 0; mode 1 (add): lane = 1 where inside, else untouched
__global__ void __launch_bounds__(VS_THREADS) view_select_kernel(CloudView cloud, uint32_t n, const __grid_constant__ FrameConsts fc,
                                                                 const uint8_t* __restrict__ mask, uint32_t mode,
                                                                 uint32_t* __restrict__ inside_count) {
    const uint32_t i = blockIdx.x * VS_THREADS + threadIdx.x;
    bool inside = false;
    if (i < n) {
        const float4 p = __ldg(cloud.pos + i);
        float pw[4], ndc[2];
        mat4_point(fc.model, p.x, p.y, p.z, pw);
        const bool visible = in_frustum(fc, pw, ndc);
        const float hw = 0.5f * fc.W, hh = 0.5f * fc.H;
        const float cx = ndc[0] * hw + hw, cy = hh - ndc[1] * hh;
        // (NaN fails every comparison)
        if (visible && cx >= 0.0f && cx < (float)fc.Wi && cy >= 0.0f && cy < (float)fc.Hi) {
            inside = __ldg(mask + (size_t)floorf(cy) * fc.Wi + (size_t)floorf(cx)) != 0;
        }
        if (mode == 0u || inside) cloud.store_visibility(i, inside ? 1.0f : 0.0f);
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, inside);
    if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(inside_count, (uint32_t)__popc(ballot));
}

void launch_view_select(CloudView cloud, uint32_t n, const FrameConsts& fc, const uint8_t* mask, uint32_t mode,
                        uint32_t* inside, cudaStream_t stream) {
    if (n == 0) return;
    view_select_kernel<<<(n + VS_THREADS - 1) / VS_THREADS, VS_THREADS, 0, stream>>>(cloud, n, fc, mask, mode, inside);
}

}  // namespace bgs
