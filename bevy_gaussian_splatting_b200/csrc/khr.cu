// khr.cu -- the decode of a KHR_gaussian_splatting glTF primitive (bgs_cloud_upload_khr; the reference's readers,
// src/io/scene.rs:1590-2015) from device copies of its accessors into the staged planes repack_kernel consumes.
//
// One thread per gaussian reads its element of every accessor (typed, strided: each span was copied as it lies in the
// file), decodes it in the reference's f32 order, and writes the gaussian's staged planes (cloud_layout.cuh): the
// position plane, the SH plane at whole chunks (padding lanes and words zero), and the rotation / scale-opacity planes
// (f32) or the packed second record (f16).  Built with -fmad=false; the normalisation is written in explicit
// __fmul_rn / __fadd_rn and exp is evaluated in f64 and rounded once, so the decode is bit for bit the oracle's.
// Each warp ORs its gaussians' rule violations and adds its zero-length quaternions into two words, read back once.
#include <cfloat>

#include "common.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int KHR_THREADS = 256;

// component i of element e (glTF component codes; the span's base and the stride keep every component aligned)
__device__ __forceinline__ float khr_component(const KhrSrc& a, uint32_t e, uint32_t i) {
    const uint8_t* p = a.data + (size_t)e * a.stride;
    switch (a.type) {
        case KHR_I8: {
            const float v = (float)reinterpret_cast<const int8_t*>(p)[i];
            return a.normalized ? fmaxf(__fdiv_rn(v, 127.0f), -1.0f) : v;
        }
        case KHR_U8: return __fdiv_rn((float)p[i], 255.0f);   // (u8 / u16 are accepted only where they read as normalised)
        case KHR_I16: {
            const float v = (float)reinterpret_cast<const int16_t*>(p)[i];
            return a.normalized ? fmaxf(__fdiv_rn(v, 32767.0f), -1.0f) : v;
        }
        case KHR_U16: return __fdiv_rn((float)reinterpret_cast<const uint16_t*>(p)[i], 65535.0f);
        default: return reinterpret_cast<const float*>(p)[i];
    }
}

__device__ __forceinline__ bool finite3(float a, float b, float c) { return isfinite(a) && isfinite(b) && isfinite(c); }

// lane l of gaussian i's SH plane: coefficient j's rgb at lanes 3j .. 3j + 2, the lanes past 3 K_d zero; without SH
// (bands 0) the DC coefficients c0 from COLOR_0 (scene.rs:1355-1362)
__device__ __forceinline__ float khr_sh_lane(const KhrDecode& k, uint32_t i, uint32_t l, const float c0[3], uint32_t& bad) {
    if (k.bands == 0) return l < 3u ? c0[l] : 0.0f;
    const uint32_t j = l / 3u;
    if (j >= k.bands) return 0.0f;
    const float v = khr_component(k.sh[j], i, l - 3u * j);
    if (!isfinite(v)) bad |= KHR_BAD_SH;
    return v;
}

template <bool F16>
__global__ void __launch_bounds__(KHR_THREADS) khr_decode_kernel(KhrDecode k, float4* __restrict__ pos, uint4* __restrict__ sh,
                                                                  uint4* __restrict__ rot, float4* __restrict__ so,
                                                                  uint32_t* __restrict__ words) {
    const uint32_t i = blockIdx.x * KHR_THREADS + threadIdx.x;
    const bool live = i < k.n;
    uint32_t bad = 0u;
    bool zero_quat = false;
    if (live) {
        const float px = khr_component(k.position, i, 0), py = khr_component(k.position, i, 1), pz = khr_component(k.position, i, 2);
        if (!finite3(px, py, pz)) bad |= KHR_BAD_POSITION;
        pos[i] = make_float4(px, py, pz, 1.0f);

        float q[4];
#pragma unroll
        for (uint32_t c = 0; c < 4; ++c) q[c] = khr_component(k.rotation, i, c);
        // normalize_quaternion (scene.rs:1979-1999): a sequential f32 sum of squares, sqrt, reciprocal, multiply
        const float l2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], q[0]), __fmul_rn(q[1], q[1])), __fmul_rn(q[2], q[2])),
                                   __fmul_rn(q[3], q[3]));
        if (l2 <= FLT_EPSILON) {
            zero_quat = true;
            q[0] = 1.0f; q[1] = 0.0f; q[2] = 0.0f; q[3] = 0.0f;
        } else {
            const float inv = __frcp_rn(__fsqrt_rn(l2));
#pragma unroll
            for (uint32_t c = 0; c < 4; ++c) q[c] = __fmul_rn(q[c], inv);
        }
        if (!finite3(q[0], q[1], q[2]) || !isfinite(q[3])) bad |= KHR_BAD_ROTATION;

        float s[3];
#pragma unroll
        for (uint32_t c = 0; c < 3; ++c) s[c] = (float)exp((double)khr_component(k.scale, i, c));
        if (!finite3(s[0], s[1], s[2])) bad |= KHR_BAD_SCALE;
        const float op = khr_component(k.opacity, i, 0);
        if (!(op >= 0.0f && op <= 1.0f)) bad |= KHR_BAD_OPACITY;

        float c0[3] = {0.0f, 0.0f, 0.0f};
        if (k.bands == 0 && k.color.data) {
#pragma unroll
            for (uint32_t c = 0; c < 3; ++c) c0[c] = khr_component(k.color, i, c);
            if (!finite3(c0[0], c0[1], c0[2])) bad |= KHR_BAD_COLOR;
#pragma unroll
            for (uint32_t c = 0; c < 3; ++c) c0[c] = __fdiv_rn(c0[c], 0.282095f);
        }
        const uint32_t units = k.sh_units;   // 16 B units of the staged SH plane per gaussian
        uint4* row = sh + (size_t)i * units;
        for (uint32_t u = 0; u < units; ++u) {
            constexpr uint32_t L = F16 ? 8u : 4u;   // lanes per unit
            float v[L];
#pragma unroll
            for (uint32_t j = 0; j < L; ++j) v[j] = khr_sh_lane(k, i, L * u + j, c0, bad);
            if constexpr (F16)   // the even coefficient in each word's low half
                row[u] = make_uint4(pack_halves(v[1], v[0]), pack_halves(v[3], v[2]), pack_halves(v[5], v[4]), pack_halves(v[7], v[6]));
            else
                row[u] = make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3]));
        }
        if constexpr (F16) {
            rot[i] = make_uint4(pack_halves(q[0], q[1]), pack_halves(q[2], q[3]), pack_halves(s[0], s[1]), pack_halves(s[2], op));
        } else {
            rot[i] = make_uint4(__float_as_uint(q[0]), __float_as_uint(q[1]), __float_as_uint(q[2]), __float_as_uint(q[3]));
            so[i] = make_float4(s[0], s[1], s[2], op);
        }
    }
    const uint32_t warp_bad = __reduce_or_sync(0xFFFFFFFFu, bad);
    const uint32_t warp_zero = __popc(__ballot_sync(0xFFFFFFFFu, zero_quat));
    if ((threadIdx.x & 31u) == 0) {
        if (warp_bad) atomicOr(&words[0], warp_bad);
        if (warp_zero) atomicAdd(&words[1], warp_zero);
    }
}

void launch_khr_decode(const KhrDecode& k, bool f16, float4* pos, void* sh, void* rot, void* so, uint32_t* words,
                       cudaStream_t stream) {
    const uint32_t grid = (k.n + KHR_THREADS - 1) / KHR_THREADS;
    if (f16)
        khr_decode_kernel<true><<<grid, KHR_THREADS, 0, stream>>>(k, pos, static_cast<uint4*>(sh), static_cast<uint4*>(rot),
                                                                   nullptr, words);
    else
        khr_decode_kernel<false><<<grid, KHR_THREADS, 0, stream>>>(k, pos, static_cast<uint4*>(sh), static_cast<uint4*>(rot),
                                                                    static_cast<float4*>(so), words);
}

}  // namespace bgs
