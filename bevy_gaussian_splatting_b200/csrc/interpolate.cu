// interpolate.cu -- two resident clouds of one size and layout blended into a third (src/morph/interpolate.rs,
// interpolate.wgsl:51-119; the reference's GaussianInterpolate { lhs, rhs }): every lane mix(l, r, t), the rotation
// normalised after it.  The factor t is the host's (cloud.cu, interpolation_factor).
//
// One thread per 16 B chunk of the output block (cloud_layout.cuh).  Each chunk is blended from the same chunk of the
// two input blocks and is self-contained: no lane reads another chunk.  The position chunk's thread also stores the
// position plane; the pad chunks are not written.  Every SH chunk is blended whole: at SH degrees below 3 that includes
// the padding lanes and, in f16, the zero words that fill the last chunk (mix(0, 0, t) = 0).
//
// Arithmetic: mix(a, b, t) = a*(1-t) + b*t (WGSL's definition, 1-t rounded once), the normalisation
// q / sqrt(((q0*q0 + q1*q1) + q2*q2) + q3*q3) in storage lane order (w, x, y, z) with (0, 0, 0, 1) when that sum is
// <= 0; every operation f32 round-to-nearest-even without FMA (explicit __fmul_rn / __fadd_rn / __fdiv_rn /
// __fsqrt_rn; the file is also built with -fmad=false), subnormals kept.  f16 halves are widened exactly and narrowed
// with round-to-nearest-even (__float2half_rn: past 65504 they become +-inf).  interpolate_oracle/ restates it (test
// infrastructure).
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

// every half of one f16 word blended on its own
__device__ __forceinline__ uint32_t mix_word(uint32_t a, uint32_t b, float t, float omt) {
    return pack_halves(mix_lane(half_hi(a), half_hi(b), t, omt), mix_lane(half_lo(a), half_lo(b), t, omt));
}

// the f16 second record of the rotation layout (encoded as planar.wgsl:306-317): the rotation normalised, the scale
// and opacity words blended half by half
__device__ __forceinline__ uint4 mix_rot_scale_opacity(uint4 a, uint4 b, float t, float omt) {
    float qa[4], qb[4];
    second_lanes(a.x, a.y, qa);
    second_lanes(b.x, b.y, qb);
    const float4 q =
        normalize_quaternion(mix4(make_float4(qa[0], qa[1], qa[2], qa[3]), make_float4(qb[0], qb[1], qb[2], qb[3]), t, omt));
    return make_uint4(pack_halves(q.x, q.y), pack_halves(q.z, q.w), mix_word(a.z, b.z, t, omt), mix_word(a.w, b.w, t, omt));
}

// the f16 second record of the covariance layout: the six entries blended, the last word written as opacity (high
// half) | +0 (encoded as planar.wgsl:286-296: pack2x16float(vec2(0.0, opacity)))
__device__ __forceinline__ uint4 mix_covariance(uint4 a, uint4 b, float t, float omt) {
    return make_uint4(mix_word(a.x, b.x, t, omt), mix_word(a.y, b.y, t, omt), mix_word(a.z, b.z, t, omt),
                      pack_halves(mix_lane(half_hi(a.w), half_hi(b.w), t, omt), 0.0f));
}

template <CloudLayout L, uint32_t D>
__global__ void __launch_bounds__(INTERP_THREADS) interpolate_kernel(const uint4* __restrict__ lhs, const uint4* __restrict__ rhs,
                                                                     size_t n_chunks, float t, CloudView out) {
    constexpr uint32_t CH = chunks(L, D);
    const size_t i = (size_t)blockIdx.x * INTERP_THREADS + threadIdx.x;
    if (i >= n_chunks) return;
    const uint32_t c = (uint32_t)(i % CH);
    if (is_pad(L, D, c)) return;
    const float omt = __fsub_rn(1.0f, t);
    const uint4 a = __ldg(lhs + i), b = __ldg(rhs + i);
    uint4 r;
    if (c == POS_CHUNK) {
        const float4 p = mix4(*reinterpret_cast<const float4*>(&a), *reinterpret_cast<const float4*>(&b), t, omt);
        r = *reinterpret_cast<const uint4*>(&p);
    } else if (is_f16(L) && c == SECOND_CHUNK) {
        r = L == CloudLayout::F16Cov ? mix_covariance(a, b, t, omt) : mix_rot_scale_opacity(a, b, t, omt);
    } else if (is_f16(L)) {
        r = make_uint4(mix_word(a.x, b.x, t, omt), mix_word(a.y, b.y, t, omt), mix_word(a.z, b.z, t, omt),
                       mix_word(a.w, b.w, t, omt));
    } else {
        float4 f = mix4(*reinterpret_cast<const float4*>(&a), *reinterpret_cast<const float4*>(&b), t, omt);
        if (c == SECOND_CHUNK) f = normalize_quaternion(f);
        r = *reinterpret_cast<const uint4*>(&f);
    }
    out.store_chunk(i / CH, c, r);
}

void launch_interpolate(CloudLayout layout, uint32_t sh_degree, CloudView lhs, CloudView rhs, uint32_t n, float t, CloudView out,
                        cudaStream_t stream) {
    const size_t n_chunks = (size_t)n * out.chunks;
    const uint32_t grid = (uint32_t)((n_chunks + INTERP_THREADS - 1) / INTERP_THREADS);
    with_layout_degree(layout, sh_degree, [&](auto L, auto D) {   // (bgs_cloud_interpolate refuses 4D clouds)
        if constexpr (!is_4d(decltype(L)::value))
            interpolate_kernel<decltype(L)::value, decltype(D)::value><<<grid, INTERP_THREADS, 0, stream>>>(lhs.blocks, rhs.blocks, n_chunks, t, out);
    });
}

}  // namespace bgs
