// subset.cu -- a resident cloud's gaussians copied into a new resident cloud (the reference's `cloud.subset(indices)`,
// src/query/select.rs:156-176), and a resident cloud read back into the planar arrays its upload call takes.
//
// Both device copies of a gaussian move unchanged: its 16 B of the position plane and its gaussian-major block
// (project.cu's repack_kernel: f16 layouts 128 B = pos | rot-scale-opacity or covariance record | 6 sh chunks, f32
// 256 B = pos | rot | scale-opacity | 12 sh chunks | pad).
//
// Selection mode (kept iff !(visibility < 0.5f), the set DrawMode::Selected draws):
//   1. subset_count_kernel: one thread per gaussian reads its position (16 B, coalesced); each warp ballots the
//      predicate into one mask word, each CTA writes its kept count;
//   2. subset_scan_kernel: one CTA turns the CTA counts into exclusive offsets and writes the total;
//   3. (host: the total is read back and the new planes are allocated)
//   4. subset_scatter_kernel: each warp walks its mask word; the kept gaussians' blocks are copied as 16 B chunks by
//      CH lanes each (f16: 8 lanes = one 128 B line, f32: 16 lanes = two), in ascending index order.
// Index mode: subset_gather_kernel copies gaussian indices[j] to j, CH threads per gaussian.
// Download: unpack_kernel is repack_kernel's inverse over one chunk of gaussians, into planar staging arrays.
#include "common.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int SUBSET_THREADS = 256;                         // 8 warps: 8 mask words per CTA
constexpr uint32_t SUBSET_WORDS_PER_CTA = SUBSET_THREADS / 32;

__device__ __forceinline__ bool subset_kept(float w) { return !(w < 0.5f); }   // NaN and +inf are kept

__global__ void __launch_bounds__(SUBSET_THREADS) subset_count_kernel(const float4* __restrict__ pos, uint32_t n,
                                                                      uint32_t* __restrict__ mask, uint32_t* __restrict__ cta_cnt) {
    __shared__ uint32_t warp_cnt[SUBSET_WORDS_PER_CTA];
    const uint32_t i = blockIdx.x * SUBSET_THREADS + threadIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const bool kept = i < n && subset_kept(__ldg(pos + i).w);
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, kept);
    if (lane == 0) {
        if (i < n) mask[i >> 5] = m;
        warp_cnt[warp] = __popc(m);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
#pragma unroll
        for (uint32_t w = 0; w < SUBSET_WORDS_PER_CTA; ++w) s += warp_cnt[w];
        cta_cnt[blockIdx.x] = s;
    }
}

// One CTA of 1024 threads: cnt[0..g) := exclusive prefix sums, *total := their sum.
__global__ void __launch_bounds__(1024) subset_scan_kernel(uint32_t* __restrict__ cnt, uint32_t g, uint32_t* __restrict__ total) {
    __shared__ uint32_t warp_sum[32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t carry = 0;
    for (uint32_t base = 0; base < g; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < g ? cnt[i] : 0u;
        uint32_t x = v;   // inclusive scan within the warp
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if ((int)lane >= d) x += y;
        }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint32_t s = warp_sum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, s, d);
                if ((int)lane >= d) s += y;
            }
            warp_sum[lane] = s;   // inclusive over the warps
        }
        __syncthreads();
        const uint32_t before = (warp ? warp_sum[warp - 1] : 0u) + x - v;
        if (i < g) cnt[i] = carry + before;
        carry += warp_sum[31];
        __syncthreads();   // (warp_sum is rewritten by the next tile)
    }
    if (threadIdx.x == 0) *total = carry;
}

// One 16 B chunk c of gaussian src's block (and, for c == 0, its position) to slot dst of the new cloud.
template <uint32_t CH>
__device__ __forceinline__ void subset_copy(const uint4* __restrict__ pos, const uint4* __restrict__ blocks, uint32_t src,
                                            uint32_t dst, uint32_t c, uint4* __restrict__ out_pos, uint4* __restrict__ out_blocks) {
    out_blocks[(size_t)dst * CH + c] = __ldg(blocks + (size_t)src * CH + c);
    if (c == 0) out_pos[dst] = __ldg(pos + src);
}

template <uint32_t CH>
__global__ void __launch_bounds__(SUBSET_THREADS) subset_scatter_kernel(const uint4* __restrict__ pos, const uint4* __restrict__ blocks,
                                                                        uint32_t n_words, const uint32_t* __restrict__ mask,
                                                                        const uint32_t* __restrict__ cta_off,
                                                                        uint4* __restrict__ out_pos, uint4* __restrict__ out_blocks) {
    constexpr uint32_t G = 32u / CH;   // gaussians per warp pass
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t word = blockIdx.x * SUBSET_WORDS_PER_CTA + warp;
    if (word >= n_words) return;       // (whole warps)
    // the slot of this word's first kept gaussian: the CTA's offset + the kept counts of the CTA's earlier words
    const uint32_t before = lane < warp ? __popc(mask[blockIdx.x * SUBSET_WORDS_PER_CTA + lane]) : 0u;
    const uint32_t base = cta_off[blockIdx.x] + __reduce_add_sync(0xFFFFFFFFu, before);
    const uint32_t m = mask[word];
    const uint32_t k = __popc(m), c = lane % CH;
    for (uint32_t j0 = 0; j0 < k; j0 += G) {
        const uint32_t j = j0 + lane / CH;
        if (j < k) subset_copy<CH>(pos, blocks, word * 32u + __fns(m, 0, (int)j + 1), base + j, c, out_pos, out_blocks);
    }
}

template <uint32_t CH>
__global__ void __launch_bounds__(SUBSET_THREADS) subset_gather_kernel(const uint4* __restrict__ pos, const uint4* __restrict__ blocks,
                                                                       const uint32_t* __restrict__ idx, uint32_t k,
                                                                       uint4* __restrict__ out_pos, uint4* __restrict__ out_blocks) {
    const size_t t = (size_t)blockIdx.x * SUBSET_THREADS + threadIdx.x;
    if (t >= (size_t)k * CH) return;
    const uint32_t j = (uint32_t)(t / CH), c = (uint32_t)(t % CH);
    subset_copy<CH>(pos, blocks, __ldg(idx + j), j, c, out_pos, out_blocks);
}

// repack_kernel's inverse over gaussians [lo, lo + m): block chunk c of gaussian lo + j goes to sh[j * SHC + k], rot[j]
// or so[j] (the position chunk and the f32 pad are skipped: the position plane is read back directly).
template <bool F16>
__global__ void __launch_bounds__(SUBSET_THREADS) unpack_kernel(const uint4* __restrict__ blocks, uint32_t lo, uint32_t m,
                                                                uint4* __restrict__ sh, uint4* __restrict__ rot, uint4* __restrict__ so) {
    constexpr uint32_t CH = F16 ? 8u : 16u, SHC = F16 ? 6u : 12u;
    const size_t t = (size_t)blockIdx.x * SUBSET_THREADS + threadIdx.x;
    if (t >= (size_t)m * CH) return;
    const uint32_t j = (uint32_t)(t / CH), c = (uint32_t)(t % CH);
    if (c == 0) return;
    const uint4 v = __ldg(blocks + (size_t)lo * CH + t);
    if (c == 1) rot[j] = v;
    else if (!F16 && c == 2) so[j] = v;
    else {
        const uint32_t k = c - (F16 ? 2u : 3u);
        if (k < SHC) sh[(size_t)j * SHC + k] = v;
    }
}

uint32_t subset_num_ctas(uint32_t n) { return (n + SUBSET_THREADS - 1) / SUBSET_THREADS; }

void launch_subset_count(const float4* pos, uint32_t n, uint32_t* mask, uint32_t* cta_cnt, uint32_t* total, cudaStream_t stream) {
    const uint32_t g = subset_num_ctas(n);
    subset_count_kernel<<<g, SUBSET_THREADS, 0, stream>>>(pos, n, mask, cta_cnt);
    subset_scan_kernel<<<1, 1024, 0, stream>>>(cta_cnt, g, total);
}

void launch_subset_scatter(bool f16, const void* pos, const void* blocks, uint32_t n, const uint32_t* mask, const uint32_t* cta_off,
                           void* out_pos, void* out_blocks, cudaStream_t stream) {
    const uint32_t g = subset_num_ctas(n), words = (n + 31) / 32;
    if (f16) subset_scatter_kernel<8><<<g, SUBSET_THREADS, 0, stream>>>((const uint4*)pos, (const uint4*)blocks, words, mask, cta_off,
                                                                         (uint4*)out_pos, (uint4*)out_blocks);
    else subset_scatter_kernel<16><<<g, SUBSET_THREADS, 0, stream>>>((const uint4*)pos, (const uint4*)blocks, words, mask, cta_off,
                                                                      (uint4*)out_pos, (uint4*)out_blocks);
}

void launch_subset_gather(bool f16, const void* pos, const void* blocks, const uint32_t* idx, uint32_t k, void* out_pos,
                          void* out_blocks, cudaStream_t stream) {
    const size_t total = (size_t)k * (f16 ? 8 : 16);
    const uint32_t grid = (uint32_t)((total + SUBSET_THREADS - 1) / SUBSET_THREADS);
    if (f16) subset_gather_kernel<8><<<grid, SUBSET_THREADS, 0, stream>>>((const uint4*)pos, (const uint4*)blocks, idx, k,
                                                                           (uint4*)out_pos, (uint4*)out_blocks);
    else subset_gather_kernel<16><<<grid, SUBSET_THREADS, 0, stream>>>((const uint4*)pos, (const uint4*)blocks, idx, k,
                                                                        (uint4*)out_pos, (uint4*)out_blocks);
}

void launch_unpack(bool f16, const void* blocks, uint32_t lo, uint32_t m, void* sh, void* rot, void* so, cudaStream_t stream) {
    const size_t total = (size_t)m * (f16 ? 8 : 16);
    const uint32_t grid = (uint32_t)((total + SUBSET_THREADS - 1) / SUBSET_THREADS);
    if (f16) unpack_kernel<true><<<grid, SUBSET_THREADS, 0, stream>>>((const uint4*)blocks, lo, m, (uint4*)sh, (uint4*)rot, (uint4*)so);
    else unpack_kernel<false><<<grid, SUBSET_THREADS, 0, stream>>>((const uint4*)blocks, lo, m, (uint4*)sh, (uint4*)rot, (uint4*)so);
}

}  // namespace bgs
