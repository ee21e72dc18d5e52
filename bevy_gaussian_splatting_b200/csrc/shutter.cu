// shutter.cu -- bgs_render_shutter's resolve: the frame from its s sub-frames' raw blended states (include/bgs.h).
//
// The shutter frame's blend (raster.cu's SubFrames variants) stores each sub-frame pixel's (C, T) as a float4, sub-frame
// after sub-frame.  One thread per pixel then sums its s states in the rule's fixed pairwise order, divides by s with
// IEEE round-to-nearest and writes the frame's pixel through the blend's own encoder (pixel.cuh's write_pixel), reading
// the target on blend-over frames.  The tree is unrolled for each s, so the s loads have addresses that depend on nothing
// but the pixel and can all be in flight before the first add; a warp's load of one sub-frame is 512 contiguous bytes.
// The pass is bandwidth-bound: s 16 B loads and one 4 / 8 / 16 B store per pixel (plus one load on blend-over frames).
#include <utility>

#include "launch.cuh"
#include "pixel.cuh"

namespace bgs {

constexpr int RESOLVE_THREADS = 256;

__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

// sum(A, B) of include/bgs.h's rule over x[i stride]: x_A when B - A == 1, else sum(A, M) + sum(M, B), M = A + (B - A + 1) / 2
// (the states are read once: streaming loads)
template <uint32_t A, uint32_t B>
__device__ __forceinline__ float4 pairwise_sum(const float4* __restrict__ x, size_t stride) {
    if constexpr (B - A == 1) {
        return __ldcs(x + A * stride);
    } else {
        constexpr uint32_t M = A + (B - A + 1) / 2;
        return add4(pairwise_sum<A, M>(x, stride), pairwise_sum<M, B>(x, stride));
    }
}

template <uint32_t S>
__global__ void __launch_bounds__(RESOLVE_THREADS)
shutter_resolve_kernel(const float4* __restrict__ sub, uint32_t wh, void* __restrict__ out, uint32_t format,
                       const uint32_t* __restrict__ truncated) {
    const uint32_t p = blockIdx.x * RESOLVE_THREADS + threadIdx.x;
    // (a truncated pair list: the blend wrote nothing and the frame is rendered again, so the target stays as it was)
    if (p >= wh || *truncated) return;
    const float4 m = pairwise_sum<0, S>(sub + p, wh);
    const float s = (float)S;
    write_pixel(out, format, p, __fdiv_rn(m.x, s), __fdiv_rn(m.y, s), __fdiv_rn(m.z, s), __fdiv_rn(m.w, s));
}

// the resolve kernels of s = 2 .. MAX_VIEWS, indexed s - 2
template <uint32_t... I>
const auto* resolve_kernels(std::integer_sequence<uint32_t, I...>) {
    static void (*const table[])(const float4*, uint32_t, void*, uint32_t, const uint32_t*) = {shutter_resolve_kernel<I + 2>...};
    return table;
}

void launch_shutter_resolve(const float4* sub, uint32_t s, uint32_t wh, void* out, uint32_t format, const uint32_t* truncated,
                            cudaStream_t stream) {
    static const auto* const kernels = resolve_kernels(std::make_integer_sequence<uint32_t, MAX_VIEWS - 1>());
    kernels[s - 2]<<<(wh + RESOLVE_THREADS - 1) / RESOLVE_THREADS, RESOLVE_THREADS, 0, stream>>>(sub, wh, out, format, truncated);
}

}  // namespace bgs
