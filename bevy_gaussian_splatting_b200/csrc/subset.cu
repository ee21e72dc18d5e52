// subset.cu -- a resident cloud's gaussians copied into a new resident cloud (the reference's `cloud.subset(indices)`,
// src/query/select.rs:156-176), and a resident cloud read back into the planar arrays its upload call takes.
//
// Both device copies of a gaussian (cloud_layout.cuh) move unchanged.
//
// Selection mode (kept iff !(visibility < 0.5f), the set DrawMode::Selected draws):
//   1. subset_count_kernel: one thread per gaussian reads its position (16 B, coalesced); each warp ballots the
//      predicate into one mask word, each CTA writes its kept count;
//   2. subset_scan_kernel: one CTA turns the CTA counts into exclusive offsets and writes the total;
//   3. (host: the total is read back and the new planes are allocated)
//   4. subset_scatter_kernel: each warp walks its mask word; the kept gaussians' blocks are copied as 16 B chunks by
//      CH lanes each (one lane per chunk), in ascending index order.
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

// One 16 B chunk c of gaussian s's block (CH chunks) to gaussian d of the new cloud (the position chunk to both copies).
template <uint32_t CH>
__device__ __forceinline__ void subset_copy(const CloudView& src, uint32_t s, uint32_t d, uint32_t c, const CloudView& dst) {
    dst.store_chunk(d, c, __ldg(src.blocks + (size_t)s * CH + c));
}

template <uint32_t CH>
__global__ void __launch_bounds__(SUBSET_THREADS) subset_scatter_kernel(CloudView src, uint32_t n_words, const uint32_t* __restrict__ mask,
                                                                        const uint32_t* __restrict__ cta_off, CloudView dst) {
    constexpr uint32_t G = 32u / CH;   // gaussians per warp pass
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t word = blockIdx.x * SUBSET_WORDS_PER_CTA + warp;
    if (word >= n_words) return;       // (whole warps)
    // the slot of this word's first kept gaussian: the CTA's offset + the kept counts of the CTA's earlier words
    const uint32_t before = lane < warp ? __popc(mask[blockIdx.x * SUBSET_WORDS_PER_CTA + lane]) : 0u;
    const uint32_t base = cta_off[blockIdx.x] + __reduce_add_sync(0xFFFFFFFFu, before);
    const uint32_t m = mask[word];
    const uint32_t k = __popc(m);
    if constexpr (G == 0) {   // (a block wider than a warp, the 4D layout's: the warp copies one gaussian at a time)
        for (uint32_t j = 0; j < k; ++j)
            for (uint32_t c = lane; c < CH; c += 32u) subset_copy<CH>(src, word * 32u + __fns(m, 0, (int)j + 1), base + j, c, dst);
    } else {
        const uint32_t c = lane % CH;
        for (uint32_t j0 = 0; j0 < k; j0 += G) {
            const uint32_t j = j0 + lane / CH;
            if (j < k) subset_copy<CH>(src, word * 32u + __fns(m, 0, (int)j + 1), base + j, c, dst);
        }
    }
}

template <uint32_t CH>
__global__ void __launch_bounds__(SUBSET_THREADS) subset_gather_kernel(CloudView src, const uint32_t* __restrict__ idx, uint32_t k,
                                                                       CloudView dst) {
    const size_t t = (size_t)blockIdx.x * SUBSET_THREADS + threadIdx.x;
    if (t >= (size_t)k * CH) return;
    const uint32_t j = (uint32_t)(t / CH), c = (uint32_t)(t % CH);
    subset_copy<CH>(src, __ldg(idx + j), j, c, dst);
}

// repack_kernel's inverse over gaussians [lo, lo + m): block chunk c of gaussian lo + j goes back to its unit of
// gaussian j in the planes (planes.pos is null: the position plane is read back directly).
template <CloudLayout L, uint32_t D>
__device__ __forceinline__ void unpack_chunk(const uint4* __restrict__ blocks, uint32_t lo, uint32_t m,
                                             const CloudPlanes<uint4>& planes, uint4* __restrict__ tt) {
    constexpr uint32_t CH = chunks(L, D);
    const size_t t = (size_t)blockIdx.x * SUBSET_THREADS + threadIdx.x;
    if (t >= (size_t)m * CH) return;
    uint4* dst = planes.unit<L, D>((uint32_t)(t % CH), t / CH, tt);
    if (dst) *dst = __ldg(blocks + (size_t)lo * CH + t);
}
template <CloudLayout L, uint32_t D>
__global__ void __launch_bounds__(SUBSET_THREADS) unpack_kernel(const uint4* __restrict__ blocks, uint32_t lo, uint32_t m,
                                                                CloudPlanes<uint4> planes) {
    unpack_chunk<L, D>(blocks, lo, m, planes, nullptr);
}
// the 4D layout's, which also writes the timestamp-timescale plane
__global__ void __launch_bounds__(SUBSET_THREADS) unpack_4d_kernel(const uint4* __restrict__ blocks, uint32_t lo, uint32_t m,
                                                                   CloudPlanes<uint4> planes, uint4* __restrict__ tt) {
    unpack_chunk<CloudLayout::F32x4D, SH_DEGREE_MAX>(blocks, lo, m, planes, tt);
}

uint32_t subset_num_ctas(uint32_t n) { return (n + SUBSET_THREADS - 1) / SUBSET_THREADS; }

void launch_subset_count(const float4* pos, uint32_t n, uint32_t* mask, uint32_t* cta_cnt, uint32_t* total, cudaStream_t stream) {
    const uint32_t g = subset_num_ctas(n);
    subset_count_kernel<<<g, SUBSET_THREADS, 0, stream>>>(pos, n, mask, cta_cnt);
    subset_scan_kernel<<<1, 1024, 0, stream>>>(cta_cnt, g, total);
}

// (the copies depend on the layout and the SH degree only through the block's size: blocks of one size run the same
// kernels, and the 4D layout's 48-chunk blocks a warp-wide variant of the scatter)
void launch_subset_scatter(CloudLayout layout, uint32_t sh_degree, CloudView src, uint32_t n, const uint32_t* mask,
                           const uint32_t* cta_off, CloudView dst, cudaStream_t stream) {
    const uint32_t g = subset_num_ctas(n), words = (n + 31) / 32;
    with_layout_degree(layout, sh_degree, [&](auto L, auto D) {
        subset_scatter_kernel<chunks(decltype(L)::value, decltype(D)::value)><<<g, SUBSET_THREADS, 0, stream>>>(src, words, mask,
                                                                                                             cta_off, dst);
    });
}

static uint32_t chunk_grid(uint32_t n, uint32_t chunks) {
    return (uint32_t)(((size_t)n * chunks + SUBSET_THREADS - 1) / SUBSET_THREADS);
}

void launch_subset_gather(CloudLayout layout, uint32_t sh_degree, CloudView src, const uint32_t* idx, uint32_t k, CloudView dst,
                          cudaStream_t stream) {
    with_layout_degree(layout, sh_degree, [&](auto L, auto D) {
        subset_gather_kernel<chunks(decltype(L)::value, decltype(D)::value)><<<chunk_grid(k, src.chunks), SUBSET_THREADS, 0, stream>>>(
            src, idx, k, dst);
    });
}

void launch_unpack(CloudLayout layout, uint32_t sh_degree, CloudView cloud, uint32_t lo, uint32_t m, void* sh, void* rot,
                   void* so, void* tt, cudaStream_t stream) {
    const CloudPlanes<uint4> planes{nullptr, static_cast<uint4*>(sh), static_cast<uint4*>(rot), static_cast<uint4*>(so)};
    const uint32_t grid = chunk_grid(m, cloud.chunks);
    with_layout_degree(layout, sh_degree, [&](auto L, auto D) {
        if constexpr (is_4d(decltype(L)::value))
            unpack_4d_kernel<<<grid, SUBSET_THREADS, 0, stream>>>(cloud.blocks, lo, m, planes, static_cast<uint4*>(tt));
        else
            unpack_kernel<decltype(L)::value, decltype(D)::value><<<grid, SUBSET_THREADS, 0, stream>>>(cloud.blocks, lo, m, planes);
    });
}

}  // namespace bgs
