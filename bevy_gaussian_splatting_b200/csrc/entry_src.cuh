// entry_src.cuh -- where a frame's entries live: one cloud (OneCloud) or a scene's segment table (SceneSrc).
//
// Key-gen, the projection, the splat depths, the depth range and the culled flags are written once over a Src.  Global
// index i of a source is gaussian i of one cloud, or gaussian i - offset of segment seg(i) of a scene, read with that
// segment's FrameConsts.  The projection's record r is entry(r) of the source's list, and the source issues the copies
// that stage its lanes' blocks.  SEGMENTED sources split their entries between launches (mine), and can list 3D clouds
// in a frame whose colour source only Gaussian4d clouds have (project_one's no_source); the kernels test the flag before
// calling mine, so that one cloud's kernels carry no trace of it.
#pragma once
#include "common.cuh"

namespace bgs {

__device__ __forceinline__ void cp_async16(uint4* dst_shared, const uint4* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_shared)), "l"(src)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Piece p of entry g sits at 16 B unit g * SCH + stage_slot<SCH>(p, g) of a warp's stage.  Stages of 8 or more chunks
// per entry: p ^ (g & 7) (a permutation of each aligned group of 8 pieces).  4-chunk stages: two entries share a 128 B
// row of banks, so p ^ ((g >> 1) & 3) -- entries g of one quarter warp take the 8 combinations of (g & 1, (g >> 1) & 3),
// hence 8 bank groups; a copy round's 8 lanes move pieces 0..3 of an even and the next odd entry, the 8 units of one row.
template <int SCH>
__device__ __forceinline__ int stage_slot(int p, int g) {
    static_assert(SCH % 8 == 0 || SCH == 4, "stages of 4 or a multiple of 8 chunks per entry");
    if constexpr (SCH == 4) return p ^ ((g >> 1) & 3);
    else return p ^ (g & 7);
}

// Src::copy<SCH, NP, BCH>: a warp's copies of pieces 0 .. NP of its 32 entries' blocks (BCH chunks each) into its
// stage, one commit group's worth: a lane's copy k moves piece (32 k + lane) % NP of entry (32 k + lane) / NP, so NP
// consecutive lanes read one block front to back.
struct OneCloud {
    const float4* pos;
    const FrameConsts& f;
    const uint4* blocks = nullptr;        // the projection's gaussian-major blocks (cloud_layout.cuh)
    const uint32_t* list = nullptr;       // the projection list: compact slot -> id (by_slot), else the far->near sort
    int by_slot = 1;
    const TemporalConsts* t = nullptr;    // Gaussian4d clouds
    static constexpr bool SEGMENTED = false;

    __device__ __forceinline__ uint32_t seg(uint32_t) const { return 0u; }
    __device__ __forceinline__ uint32_t advance(uint32_t j, uint32_t) const { return j; }
    __device__ __forceinline__ bool mine(uint32_t) const { return true; }
    __device__ __forceinline__ const FrameConsts& fc(uint32_t) const { return f; }
    __device__ __forceinline__ const TemporalConsts& tc(uint32_t) const { return *t; }
    __device__ __forceinline__ const float4* pos_at(uint32_t, uint32_t i) const { return pos + i; }
    template <int BCH>
    __device__ __forceinline__ const uint4* block_at(uint32_t, uint32_t i) const { return blocks + (size_t)i * BCH; }
    // record r's gaussian id (0 past the list's end)
    __device__ __forceinline__ uint32_t entry(uint32_t r, uint32_t n_vis) const {
        return n_vis > r ? (by_slot ? __ldg(list + r) : __ldg(list + (n_vis - 1u - r))) : 0u;
    }
    // the lanes shuffle their 32-bit ids; entries g >= n_valid (past the list's end) copy nothing
    template <int SCH, int NP, int BCH>
    __device__ __forceinline__ void copy(uint32_t id, uint32_t n_valid, uint4* stage, int lane) const {
        static_assert(32 % NP == 0 && NP <= SCH, "NP lanes per block");
#pragma unroll
        for (int k = 0; k < NP; ++k) {
            const int g = (32 * k + lane) / NP, p = lane % NP;
            const uint32_t gid = __shfl_sync(0xFFFFFFFFu, id, g);
            if ((uint32_t)g < n_valid) cp_async16(stage + g * SCH + stage_slot<SCH>(p, g), block_at<BCH>(0u, gid) + p);
        }
    }
};

// A segment table: bgs_render_scene's (SceneTable, a kernel parameter; SceneSrc) or bgs_render_entities_many's
// (SceneTableDev, in device memory; SceneSrcDev).  `groups` has bit b set for the segments of project_group b this launch
// covers; `times` are the per-segment times of Gaussian4d segments.  seg / advance give the segment of an index (seg clamps
// one past the end to the last gaussian's segment; advance walks forward from j for an index that only grows within a
// thread).
template <class Table>
struct SegmentSrc {
    const Table& t;
    uint32_t groups = ~0u;
    const uint32_t* slot_ids = nullptr;   // compact slot -> global index
    const TemporalConsts* times = nullptr;
    static constexpr bool SEGMENTED = true;
    static constexpr uint32_t NONE = 0xFFFFFFFFu;

    __device__ __forceinline__ uint32_t seg(uint32_t i) const { return t.find(i < t.n_total ? i : t.n_total - 1u); }
    __device__ __forceinline__ uint32_t advance(uint32_t j, uint32_t i) const { return t.advance(j, i); }
    __device__ __forceinline__ bool mine(uint32_t j) const { return (groups >> t.seg[j].group) & 1u; }
    __device__ __forceinline__ const FrameConsts& fc(uint32_t j) const { return t.seg[j].fc; }
    __device__ __forceinline__ const TemporalConsts& tc(uint32_t j) const { return times[j]; }
    __device__ __forceinline__ const float4* pos_at(uint32_t j, uint32_t i) const { return t.seg[j].pos + (i - t.seg[j].offset); }
    template <int BCH>
    __device__ __forceinline__ const uint4* block_at(uint32_t j, uint32_t i) const {
        return static_cast<const uint4*>(t.seg[j].blocks) + (size_t)(i - t.seg[j].offset) * BCH;
    }
    // record r's global index (NONE past the list's end)
    __device__ __forceinline__ uint32_t entry(uint32_t r, uint32_t n_vis) const { return r < n_vis ? __ldg(slot_ids + r) : NONE; }
    // the lanes shuffle their 64-bit block pointers, null past the list's end or for another launch's segment
    template <int SCH, int NP, int BCH>
    __device__ __forceinline__ void copy(uint32_t i, uint32_t, uint4* stage, int lane) const {
        static_assert(32 % NP == 0 && NP <= SCH, "NP lanes per block");
        const uint4* block = nullptr;
        if (i != NONE) {
            const uint32_t j = seg(i);
            if (mine(j)) block = block_at<BCH>(j, i);
        }
#pragma unroll
        for (int k = 0; k < NP; ++k) {
            const int g = (32 * k + lane) / NP, p = lane % NP;
            const uint4* src = reinterpret_cast<const uint4*>(
                __shfl_sync(0xFFFFFFFFu, (unsigned long long)reinterpret_cast<uintptr_t>(block), g));
            if (src) cp_async16(stage + g * SCH + stage_slot<SCH>(p, g), src + p);
        }
    }
};
using SceneSrc = SegmentSrc<SceneTable>;
using SceneSrcDev = SegmentSrc<SceneTableDev>;

// The grid of a persistent grid-stride kernel over entries whose count only the device knows: ceil(n_hint / threads)
// CTAs, at most ctas_per_sm per SM, at least one.
inline uint32_t persistent_grid(uint32_t n_hint, int threads, int ctas_per_sm, int sm_count) {
    uint32_t grid = (n_hint + threads - 1) / threads;
    if (grid > (uint32_t)(ctas_per_sm * sm_count)) grid = (uint32_t)(ctas_per_sm * sm_count);
    if (grid < 1u) grid = 1u;
    return grid;
}

}  // namespace bgs
