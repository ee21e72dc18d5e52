// cloud_layout.cuh -- how a resident cloud is stored on the device.  Every kernel and host call that reads or writes a
// cloud's storage takes its layout facts from here.
//
// A cloud is stored twice:
//  * the position plane: 16 B per gaussian (x, y, z, visibility), the only array key-gen streams;
//  * the gaussian-major blocks, made once at upload (repack_kernel) and gathered by the projection, so that a visible
//    splat touches only its own line(s).  A block is a row of 16 B chunks; its size depends on the layout and on the SH
//    degree d (include/bgs.h: S_d = 4, 12, 28, 48 floats for d = 0..3):
//      f16 layouts, d 3: 128 B: position | second record | 6 SH chunks
//                   d 2: 128 B: position | second record | 4 SH chunks (14 words, 2 zero) | 2 pad
//                   d 1:  64 B: position | second record | 2 SH chunks (6 words, 2 zero)
//                   d 0:  64 B: position | second record | 1 SH chunk (2 words, 2 zero) | 1 pad
//      f32,         d 3: 256 B: position | rotation | scale-opacity | 12 SH chunks | pad
//                   d 2: 256 B: position | rotation | scale-opacity | 7 SH chunks | 6 pad
//                   d 1: 128 B: position | rotation | scale-opacity | 3 SH chunks | 2 pad
//                   d 0:  64 B: position | rotation | scale-opacity | 1 SH chunk
//      f32 4D,      768 B: position | rotation | rotation_r | scale-opacity | timestamp-timescale | 36 SH chunks | 7 pad
//    Blocks are 4, 8, 16 or 48 chunks, so a whole number of them fills a 128 B line and a warp's 32 lanes copy a block
//    in whole rounds (entry_src.cuh: Src::copy).  (f32 d 2 would fit 160 B, but a 10-chunk block breaks both.)
//    (4D: the five geometry chunks and the first three SH chunks fill the first 128 B line, the only one the projection
//    stages; the coefficients are fetched only for drawn splats of the colour sources that read them)
//    The f16 second record is the packed rotation-scale-opacity words or, in the covariance layout, the
//    Covariance3dOpacityPacked128 record.
// The position and the visibility lane therefore live in both copies.  Every write of them goes through CloudView's
// stores, which update both.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>

#include "common.cuh"

namespace bgs {

// bgs_cloud_upload_f32, _f16, _f16_cov (whose second record holds the precomputed covariance) and _4d (Gaussian4d: two
// rotations, a timestamp and a timescale, spherindrical coefficients; f32 only)
enum class CloudLayout : uint32_t { F32, F16, F16Cov, F32x4D };

__host__ __device__ constexpr bool is_f16(CloudLayout l) { return l == CloudLayout::F16 || l == CloudLayout::F16Cov; }
__host__ __device__ constexpr bool is_4d(CloudLayout l) { return l == CloudLayout::F32x4D; }

// ---- the SH degree (include/bgs.h): K_d = (d + 1)^2 coefficients per channel, S_d = pad4(3 K_d) floats per gaussian,
// coefficient k of channel c at sh[3 k + c]; lanes 3 K_d .. S_d - 1 are padding (stored, never evaluated).  4D clouds
// are degree 3.
constexpr uint32_t SH_DEGREE_MAX = 3;
__host__ __device__ constexpr uint32_t sh_bands(uint32_t d) { return (d + 1) * (d + 1); }
__host__ __device__ constexpr uint32_t sh_floats(uint32_t d) { return d == 0 ? 4u : d == 1 ? 12u : d == 2 ? 28u : 48u; }

// ---- the block: 16 B chunks and the role of each
__host__ __device__ constexpr uint32_t chunks(CloudLayout l, uint32_t d) {
    return is_4d(l) ? 48u : is_f16(l) ? (d <= 1 ? 4u : 8u) : (d == 0 ? 4u : d == 1 ? 8u : 16u);
}
__host__ __device__ constexpr size_t block_bytes(CloudLayout l, uint32_t d) { return (size_t)chunks(l, d) * 16u; }
constexpr uint32_t POS_CHUNK = 0;      // position and visibility, as in the position plane
constexpr uint32_t SECOND_CHUNK = 1;   // f16: the second record; f32 and 4D: the rotation (w, x, y, z)
constexpr uint32_t SO_CHUNK = 2;       // f32 only: scale and opacity
constexpr uint32_t ROT_R_CHUNK = 2;    // 4D: the right rotation rotation_r (w, x, y, z)
constexpr uint32_t SO_4D_CHUNK = 3;    // 4D: scale and opacity
constexpr uint32_t TT_CHUNK = 4;       // 4D: timestamp, timescale, pad, pad
__host__ __device__ constexpr uint32_t sh_first(CloudLayout l) { return is_4d(l) ? 5u : is_f16(l) ? 2u : 3u; }
// the SH plane of one gaussian as the upload and download calls take it: S_d floats (f32), S_d / 2 words (f16)
__host__ __device__ constexpr size_t sh_plane_bytes(CloudLayout l, uint32_t d) {
    return is_4d(l) ? 576u : is_f16(l) ? (size_t)sh_floats(d) * 2u : (size_t)sh_floats(d) * 4u;
}
// ... and the 16 B chunks it occupies in the block (f16 d < 3: the last chunk's unused words are zero)
__host__ __device__ constexpr uint32_t sh_chunks(CloudLayout l, uint32_t d) { return (uint32_t)((sh_plane_bytes(l, d) + 15u) / 16u); }
// chunks from sh_first + sh_chunks to the block's end are padding (f32 d 3: chunk 15, 4D: 41..47), never read or written
__host__ __device__ constexpr bool is_pad(CloudLayout l, uint32_t d, uint32_t c) { return c >= sh_first(l) + sh_chunks(l, d); }

// ---- the planar arrays the upload and download calls take (include/bgs.h), in this order
enum : int {
    PLANE_POS, PLANE_SH, PLANE_ROT /* f16: the second record; 4D: rotation | rotation_r */, PLANE_SO /* f32 and 4D */,
    PLANE_TT /* 4D only: timestamp_timescale */, PLANES
};
// bytes per gaussian of plane p in the caller's arrays
__host__ __device__ constexpr size_t plane_bytes(CloudLayout l, uint32_t d, int p) {
    return p == PLANE_SH ? sh_plane_bytes(l, d)
           : p == PLANE_ROT ? (is_4d(l) ? 32u : 16u)
           : (p == PLANE_SO && is_f16(l)) || (p == PLANE_TT && !is_4d(l)) ? 0u : 16u;
}
// ... and in device staging, where every gaussian's SH plane fills whole chunks (the repack and unpack read and write
// 16 B units)
__host__ __device__ constexpr size_t staged_bytes(CloudLayout l, uint32_t d, int p) {
    return p == PLANE_SH ? (size_t)sh_chunks(l, d) * 16u : plane_bytes(l, d, p);
}
__host__ __device__ constexpr size_t planar_bytes(CloudLayout l, uint32_t d) {
    return plane_bytes(l, d, PLANE_POS) + plane_bytes(l, d, PLANE_SH) + plane_bytes(l, d, PLANE_ROT) +
           plane_bytes(l, d, PLANE_SO) + plane_bytes(l, d, PLANE_TT);
}

// The staged planes in 16 B units (U: uint4 or const uint4).  unit() is the one chunk-to-plane map: the upload's repack reads
// chunk c of gaussian i's block from it, the download's unpack writes the chunk back to it, so the two are inverses.
// Null for the padding and for a null plane (the download reads the position plane directly).  The 4D layout's
// timestamp-timescale plane `tt` travels beside the struct (a trailing kernel argument), so that the arguments of the
// other layouts' kernels keep their offsets.
template <class U>
struct CloudPlanes {
    U *pos, *sh, *rot, *so;
    template <CloudLayout L, uint32_t D>
    __device__ __forceinline__ U* unit(uint32_t c, size_t i, U* tt = nullptr) const {
        if (c == POS_CHUNK) return pos ? pos + i : nullptr;
        if constexpr (is_4d(L)) {
            if (c == SECOND_CHUNK || c == ROT_R_CHUNK) return rot + 2 * i + (c - SECOND_CHUNK);
            if (c == SO_4D_CHUNK) return so + i;
            if (c == TT_CHUNK) return tt + i;
        } else {
            if (c == SECOND_CHUNK) return rot + i;
            if (!is_f16(L) && c == SO_CHUNK) return so + i;
        }
        return is_pad(L, D, c) ? nullptr : sh + i * sh_chunks(L, D) + (c - sh_first(L));
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
    else if (l == CloudLayout::F16Cov) f(std::integral_constant<CloudLayout, CloudLayout::F16Cov>{});
    else f(std::integral_constant<CloudLayout, CloudLayout::F32x4D>{});
}

// f(layout tag, degree tag): the launch of a kernel templated on the layout and the SH degree (4D clouds: degree 3)
template <class F>
void with_layout_degree(CloudLayout l, uint32_t d, F f) {
    with_layout(l, [&](auto L) {
        using D0 = std::integral_constant<uint32_t, 0>;
        using D1 = std::integral_constant<uint32_t, 1>;
        using D2 = std::integral_constant<uint32_t, 2>;
        using D3 = std::integral_constant<uint32_t, 3>;
        if constexpr (is_4d(decltype(L)::value)) f(L, D3{});
        else if (d == 0) f(L, D0{});
        else if (d == 1) f(L, D1{});
        else if (d == 2) f(L, D2{});
        else f(L, D3{});
    });
}

}  // namespace bgs
