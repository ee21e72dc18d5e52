// cloud_layout.cuh -- how a resident cloud is stored on the device.  Every kernel and host call that reads or writes a
// cloud's storage takes its layout facts from here.
//
// A cloud is stored twice:
//  * the position plane: 16 B per gaussian (x, y, z, visibility), the only array key-gen streams;
//  * the gaussian-major blocks, made once at upload (repack_kernel) and gathered by the projection, so that a visible
//    splat touches only its own line(s).  A block is a row of 16 B chunks:
//      f16 layouts, 128 B: position | second record | 6 SH chunks
//      f32,         256 B: position | rotation | scale-opacity | 12 SH chunks | pad
//    The f16 second record is the packed rotation-scale-opacity words or, in the covariance layout, the
//    Covariance3dOpacityPacked128 record.
// The position and the visibility lane therefore live in both copies.  Every write of them goes through CloudView's
// stores, which update both.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>

#include "common.cuh"

namespace bgs {

// bgs_cloud_upload_f32, _f16 and _f16_cov (whose second record holds the precomputed covariance)
enum class CloudLayout : uint32_t { F32, F16, F16Cov };

__host__ __device__ constexpr bool is_f16(CloudLayout l) { return l != CloudLayout::F32; }

// ---- the block: 16 B chunks and the role of each
__host__ __device__ constexpr uint32_t chunks(CloudLayout l) { return is_f16(l) ? 8u : 16u; }
__host__ __device__ constexpr size_t block_bytes(CloudLayout l) { return (size_t)chunks(l) * 16u; }
constexpr uint32_t POS_CHUNK = 0;      // position and visibility, as in the position plane
constexpr uint32_t SECOND_CHUNK = 1;   // f16: the second record; f32: the rotation (w, x, y, z)
constexpr uint32_t SO_CHUNK = 2;       // f32 only: scale and opacity
__host__ __device__ constexpr uint32_t sh_first(CloudLayout l) { return is_f16(l) ? 2u : 3u; }
__host__ __device__ constexpr uint32_t sh_chunks(CloudLayout l) { return is_f16(l) ? 6u : 12u; }
// chunks from sh_first + sh_chunks to the block's end are padding (f32: chunk 15), never read or written
__host__ __device__ constexpr bool is_pad(CloudLayout l, uint32_t c) { return c >= sh_first(l) + sh_chunks(l); }

// ---- the planar arrays the upload and download calls take (include/bgs.h), in this order
enum : int { PLANE_POS, PLANE_SH, PLANE_ROT /* f16: the second record */, PLANE_SO /* f32 only */, PLANES };
__host__ __device__ constexpr size_t plane_bytes(CloudLayout l, int p) {
    return p == PLANE_SH ? (size_t)sh_chunks(l) * 16u : (p == PLANE_SO && is_f16(l)) ? 0u : 16u;
}
__host__ __device__ constexpr size_t planar_bytes(CloudLayout l) {
    return plane_bytes(l, PLANE_POS) + plane_bytes(l, PLANE_SH) + plane_bytes(l, PLANE_ROT) + plane_bytes(l, PLANE_SO);
}

// The planes in 16 B units (U: uint4 or const uint4).  unit() is the one chunk-to-plane map: the upload's repack reads
// chunk c of gaussian i's block from it, the download's unpack writes the chunk back to it, so the two are inverses.
// Null for the padding and for a null plane (the download reads the position plane directly).
template <class U>
struct CloudPlanes {
    U *pos, *sh, *rot, *so;
    template <CloudLayout L>
    __device__ __forceinline__ U* unit(uint32_t c, size_t i) const {
        if (c == POS_CHUNK) return pos ? pos + i : nullptr;
        if (c == SECOND_CHUNK) return rot + i;
        if (!is_f16(L) && c == SO_CHUNK) return so + i;
        return is_pad(L, c) ? nullptr : sh + i * sh_chunks(L) + (c - sh_first(L));
    }
};

// ---- f16 words: two halves each
__device__ __forceinline__ float half_lo(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w & 0xFFFFu))); }
__device__ __forceinline__ float half_hi(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }
// round to nearest even (past 65504: +-inf)
__device__ __forceinline__ uint32_t pack_halves(float hi, float lo) {
    return ((uint32_t)__half_as_ushort(__float2half_rn(hi)) << 16) | (uint32_t)__half_as_ushort(__float2half_rn(lo));
}
// Two words of the f16 second record as four lanes, high half first: words x, y are the rotation (w, x | y, z), words
// z, w are scale x, y | scale z, opacity (planar.wgsl:154-176).  The covariance record occupies the same lanes:
// c0, c1 | c2, c3 | c4, c5 | opacity in the high half (planar.wgsl:133-152).  SH words hold their coefficients low half
// first.
__device__ __forceinline__ void second_lanes(uint32_t a, uint32_t b, float out[4]) {
    out[0] = half_hi(a); out[1] = half_lo(a); out[2] = half_hi(b); out[3] = half_lo(b);
}

// ---- a cloud's storage as the kernels that write it see it
struct CloudView {
    float4* pos;       // the position plane
    uint4* blocks;     // the gaussian-major blocks
    uint32_t chunks;   // 16 B chunks per block
    __device__ __forceinline__ void store_position(size_t i, float4 p) const {
        pos[i] = p;
        reinterpret_cast<float4*>(blocks)[i * chunks + POS_CHUNK] = p;
    }
    __device__ __forceinline__ void store_visibility(size_t i, float v) const {
        pos[i].w = v;
        reinterpret_cast<float4*>(blocks)[i * chunks + POS_CHUNK].w = v;
    }
    // chunk c of gaussian i's block, for kernels with one thread per chunk.  All lanes store their chunks with one
    // instruction: storing the position chunk on a branch of its own split that store and made the f32 interpolation
    // 9 % slower (H100 80GB HBM3, 700 W)
    __device__ __forceinline__ void store_chunk(size_t i, uint32_t c, uint4 v) const {
        blocks[i * chunks + c] = v;
        if (c == POS_CHUNK) pos[i] = *reinterpret_cast<const float4*>(&v);
    }
};

// f(tag) with decltype(tag)::value == l: the launch of a kernel templated on the layout
template <class F>
void with_layout(CloudLayout l, F f) {
    if (l == CloudLayout::F32) f(std::integral_constant<CloudLayout, CloudLayout::F32>{});
    else if (l == CloudLayout::F16) f(std::integral_constant<CloudLayout, CloudLayout::F16>{});
    else f(std::integral_constant<CloudLayout, CloudLayout::F16Cov>{});
}

}  // namespace bgs
