// interpolate.cu -- two resident clouds of one size and layout blended into a third (src/morph/interpolate.rs,
// interpolate.wgsl:51-119; the reference's GaussianInterpolate { lhs, rhs }): every lane mix(l, r, t), the rotation
// normalised after it.  The factor t is the host's (cloud.cu, interpolation_factor).
//
// One thread per 16 B chunk of the output block (project.cu's repack_kernel layout: f16 layouts 128 B = pos |
// rot-scale-opacity or covariance record | 6 sh chunks, f32 256 B = pos | rot | scale-opacity | 12 sh chunks | pad).
// Each chunk is blended from the same chunk of the two input blocks and is self-contained: no lane reads another
// chunk.  The chunk-0 thread also stores the position plane; the f32 pad chunk is not written.
//
// Arithmetic: mix(a, b, t) = a*(1-t) + b*t (WGSL's definition, 1-t rounded once), the normalisation
// q / sqrt(((q0*q0 + q1*q1) + q2*q2) + q3*q3) in storage lane order (w, x, y, z) with (0, 0, 0, 1) when that sum is
// <= 0; every operation f32 round-to-nearest-even without FMA (explicit __fmul_rn / __fadd_rn / __fdiv_rn /
// __fsqrt_rn; the file is also built with -fmad=false), subnormals kept.  f16 halves are widened exactly and narrowed
// with round-to-nearest-even (__float2half_rn: past 65504 they become +-inf).  interpolate_oracle/ restates it (test
// infrastructure).
#include <cuda_fp16.h>

#include "common.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int INTERP_THREADS = 256;

__device__ __forceinline__ float mix_lane(float a, float b, float t, float omt) {
    return __fadd_rn(__fmul_rn(a, omt), __fmul_rn(b, t));
}

__device__ __forceinline__ float4 mix4(float4 a, float4 b, float t, float omt) {
    return make_float4(mix_lane(a.x, b.x, t, omt), mix_lane(a.y, b.y, t, omt), mix_lane(a.z, b.z, t, omt),
                       mix_lane(a.w, b.w, t, omt));
}

// interpolate.wgsl:59-65, q = (w, x, y, z) in storage order
__device__ __forceinline__ float4 normalize_quaternion(float4 q) {
    const float l2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.x, q.x), __fmul_rn(q.y, q.y)), __fmul_rn(q.z, q.z)),
                               __fmul_rn(q.w, q.w));
    if (l2 <= 0.0f) return make_float4(0.0f, 0.0f, 0.0f, 1.0f);
    const float s = __fsqrt_rn(l2);
    return make_float4(__fdiv_rn(q.x, s), __fdiv_rn(q.y, s), __fdiv_rn(q.z, s), __fdiv_rn(q.w, s));
}

__device__ __forceinline__ float lo_half(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w & 0xFFFFu))); }
__device__ __forceinline__ float hi_half(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }
__device__ __forceinline__ uint32_t pack_halves(float hi, float lo) {
    return ((uint32_t)__half_as_ushort(__float2half_rn(hi)) << 16) | (uint32_t)__half_as_ushort(__float2half_rn(lo));
}

// every half of one f16 word blended on its own
__device__ __forceinline__ uint32_t mix_word(uint32_t a, uint32_t b, float t, float omt) {
    return pack_halves(mix_lane(hi_half(a), hi_half(b), t, omt), mix_lane(lo_half(a), lo_half(b), t, omt));
}

// f16 chunk 1 of the rotation layout: words x, y = rotation (w = hi x, x = lo x, y = hi y, z = lo y), words z, w =
// scale.x | scale.y, scale.z | opacity (planar.wgsl:154-176, encoded as :306-317)
__device__ __forceinline__ uint4 mix_rot_scale_opacity(uint4 a, uint4 b, float t, float omt) {
    const float4 qa = make_float4(hi_half(a.x), lo_half(a.x), hi_half(a.y), lo_half(a.y));
    const float4 qb = make_float4(hi_half(b.x), lo_half(b.x), hi_half(b.y), lo_half(b.y));
    const float4 q = normalize_quaternion(mix4(qa, qb, t, omt));
    return make_uint4(pack_halves(q.x, q.y), pack_halves(q.z, q.w), mix_word(a.z, b.z, t, omt), mix_word(a.w, b.w, t, omt));
}

// f16 chunk 1 of the covariance layout: words x, y, z = the six entries, word w = opacity (hi) | +0 (lo)
// (planar.wgsl:133-152, encoded as :286-296: pack2x16float(vec2(0.0, opacity)))
__device__ __forceinline__ uint4 mix_covariance(uint4 a, uint4 b, float t, float omt) {
    return make_uint4(mix_word(a.x, b.x, t, omt), mix_word(a.y, b.y, t, omt), mix_word(a.z, b.z, t, omt),
                      pack_halves(mix_lane(hi_half(a.w), hi_half(b.w), t, omt), 0.0f));
}

template <bool F16, bool COV>
__global__ void __launch_bounds__(INTERP_THREADS) interpolate_kernel(const uint4* __restrict__ lhs, const uint4* __restrict__ rhs,
                                                                     size_t chunks, float t, uint4* __restrict__ out_blocks,
                                                                     float4* __restrict__ out_pos) {
    constexpr uint32_t CH = F16 ? 8u : 16u;
    const size_t i = (size_t)blockIdx.x * INTERP_THREADS + threadIdx.x;
    if (i >= chunks) return;
    const uint32_t c = (uint32_t)(i % CH);
    if (!F16 && c == 15) return;   // f32 pad
    const float omt = __fsub_rn(1.0f, t);
    const uint4 a = __ldg(lhs + i), b = __ldg(rhs + i);
    uint4 r;
    if (c == 0) {
        const float4 p = mix4(*reinterpret_cast<const float4*>(&a), *reinterpret_cast<const float4*>(&b), t, omt);
        out_pos[i / CH] = p;
        r = *reinterpret_cast<const uint4*>(&p);
    } else if (F16 && c == 1) {
        r = COV ? mix_covariance(a, b, t, omt) : mix_rot_scale_opacity(a, b, t, omt);
    } else if (F16) {
        r = make_uint4(mix_word(a.x, b.x, t, omt), mix_word(a.y, b.y, t, omt), mix_word(a.z, b.z, t, omt),
                       mix_word(a.w, b.w, t, omt));
    } else {
        float4 f = mix4(*reinterpret_cast<const float4*>(&a), *reinterpret_cast<const float4*>(&b), t, omt);
        if (c == 1) f = normalize_quaternion(f);
        r = *reinterpret_cast<const uint4*>(&f);
    }
    out_blocks[i] = r;
}

void launch_interpolate(bool f16, bool cov, const void* lhs_blocks, const void* rhs_blocks, uint32_t n, float t,
                        void* out_blocks, float4* out_pos, cudaStream_t stream) {
    const size_t chunks = (size_t)n * (f16 ? 8 : 16);
    const uint32_t grid = (uint32_t)((chunks + INTERP_THREADS - 1) / INTERP_THREADS);
    const uint4* l = static_cast<const uint4*>(lhs_blocks);
    const uint4* r = static_cast<const uint4*>(rhs_blocks);
    uint4* o = static_cast<uint4*>(out_blocks);
    if (!f16) interpolate_kernel<false, false><<<grid, INTERP_THREADS, 0, stream>>>(l, r, chunks, t, o, out_pos);
    else if (cov) interpolate_kernel<true, true><<<grid, INTERP_THREADS, 0, stream>>>(l, r, chunks, t, o, out_pos);
    else interpolate_kernel<true, false><<<grid, INTERP_THREADS, 0, stream>>>(l, r, chunks, t, o, out_pos);
}

}  // namespace bgs
