// select.cu -- SparseSelect (src/query/sparse.rs:24-54) on the device-resident cloud: the neighbour count of every
// gaussian within a fixed radius, and the visibility lane it decides.
//
// The reference builds a kd-tree over every position and selects gaussian i when
// tree.within_radius(p_i, radius).len() < neighbor_threshold.  Here the same fixed-radius query runs on a hashed
// uniform grid:
//   1. select_keys_kernel: key = hashed bucket of the gaussian's cell (cells slightly larger than the radius, so
//      every accepted pair lies in cells at most one apart on each axis); non-finite positions get the sentinel key
//      n_buckets, which sorts last and which no lookup visits;
//   2. the stable radix sort of radix.cu over (key, index), whose `ranges` epilogue yields each bucket's slice;
//   3. select_gather_kernel: positions in bucket order, so each bucket's scan reads contiguous memory;
//   4. select_count_kernel: one thread per sorted entry (neighbouring threads share cells) scans the distinct
//      buckets of its 27 neighbour cells with the exact f32 test, stops once the count reaches the threshold,
//      and writes the visibility into both device copies (position plane .w, gaussian-major block .w).
// Hash collisions only add distance tests; the dedupe of the 27 buckets keeps a bucket from being counted twice.
//
// Cost: O(N) for keys and sort; the count is O(N x min(threshold, neighbours in 27 cells)), plus the collisions.
// Worst case: a radius that puts most of the cloud into one cell (or one clamped cell, see cell_coord) with a large
// threshold is O(N x threshold).
#include "common.cuh"

namespace bgs {

// The cell / bucket functions.  select_oracle/select_oracle.cpp restates them (test infrastructure).
// Cell coordinate of a coordinate p: floor(p / cell) in f64, clamped to +-2^40 (below that the two f64 quotients of
// an accepted pair are off by at most 2^-12 together, well inside the 2^-10 margin of the cell size).  Clamping is
// monotone, so it only merges cells.
constexpr double SEL_CLAMP = 1099511627776.0;   // 2^40
__host__ __device__ __forceinline__ long long sel_cell_coord(float p, double cell) {
    double q = (double)p / cell;
    q = q < -SEL_CLAMP ? -SEL_CLAMP : (q > SEL_CLAMP ? SEL_CLAMP : q);
    return (long long)floor(q);
}
// The cell size: the radius widened by 2^-10 in f64, so the true distance of any pair the f32 test accepts (a few
// ulps above the radius at most) stays below one cell.
__host__ __device__ __forceinline__ double sel_cell_size(float radius) { return (double)radius * (1.0 + 1.0 / 1024.0); }
constexpr unsigned long long SEL_HX = 0x9E3779B97F4A7C15ull, SEL_HY = 0xC2B2AE3D27D4EB4Full, SEL_HZ = 0x165667B19E3779F9ull;
// the linear part of the hash: neighbour cells differ from it by (dx * HX + dy * HY + dz * HZ) mod 2^64
__host__ __device__ __forceinline__ unsigned long long sel_cell_lin(long long cx, long long cy, long long cz) {
    return (unsigned long long)cx * SEL_HX + (unsigned long long)cy * SEL_HY + (unsigned long long)cz * SEL_HZ;
}
__host__ __device__ __forceinline__ uint32_t sel_bucket(unsigned long long h, uint32_t bucket_mask) {
    h ^= h >> 29;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 32;
    return (uint32_t)h & bucket_mask;
}
__device__ __forceinline__ bool sel_finite(float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

constexpr int SEL_THREADS = 256;

__global__ void __launch_bounds__(SEL_THREADS) select_keys_kernel(const float4* __restrict__ pos, uint32_t n, double cell,
                                                                  uint32_t n_buckets, uint32_t* __restrict__ keys,
                                                                  uint32_t* __restrict__ vals, uint32_t* __restrict__ n_sort) {
    const uint32_t i = blockIdx.x * SEL_THREADS + threadIdx.x;
    if (i == 0) *n_sort = n;
    if (i >= n) return;
    const float4 p = __ldg(pos + i);
    uint32_t k = n_buckets;   // sentinel: sorts after every bucket, never looked up
    if (sel_finite(p))
        k = sel_bucket(sel_cell_lin(sel_cell_coord(p.x, cell), sel_cell_coord(p.y, cell), sel_cell_coord(p.z, cell)),
                       n_buckets - 1u);
    keys[i] = k;
    vals[i] = i;
}

__global__ void __launch_bounds__(SEL_THREADS) select_gather_kernel(const float4* __restrict__ pos, const uint32_t* __restrict__ ids,
                                                                    uint32_t n, float4* __restrict__ spos) {
    const uint32_t t = blockIdx.x * SEL_THREADS + threadIdx.x;
    if (t < n) spos[t] = __ldg(pos + __ldg(ids + t));
}

// One thread per sorted entry t (gaussian ids[t], position spos[t]).  count = #{j : d2(i, j) < r2}, j == i included,
// d2 = ((dx*dx + dy*dy) + dz*dz), every operation f32 round-to-nearest-even without contraction.
__global__ void __launch_bounds__(SEL_THREADS) select_count_kernel(const float4* __restrict__ spos, const uint32_t* __restrict__ ids,
                                                                   const uint2* __restrict__ ranges, uint32_t n, double cell,
                                                                   uint32_t bucket_mask, float r2, uint32_t threshold,
                                                                   float* __restrict__ pos_w, float* __restrict__ block_w,
                                                                   uint32_t block_stride, uint32_t* __restrict__ selected) {
    const uint32_t t = blockIdx.x * SEL_THREADS + threadIdx.x;
    bool sel = false;
    if (t < n) {
        const float4 p = spos[t];
        uint32_t cnt = 0u;
        if (sel_finite(p) && threshold > 0u) {   // (a non-finite position has a NaN d2 against everything: count 0)
            const long long cx = sel_cell_coord(p.x, cell), cy = sel_cell_coord(p.y, cell), cz = sel_cell_coord(p.z, cell);
            const unsigned long long h0 = sel_cell_lin(cx - 1, cy - 1, cz - 1);
            uint32_t b[27];
#pragma unroll
            for (int k = 0; k < 27; ++k)
                b[k] = sel_bucket(h0 + (unsigned long long)(k % 3) * SEL_HX + (unsigned long long)(k / 3 % 3) * SEL_HY +
                                      (unsigned long long)(k / 9) * SEL_HZ, bucket_mask);
#pragma unroll
            for (int k = 0; k < 27; ++k) {
                // two of the 27 cells may hash to one bucket: scan it once
                bool dup = false;
#pragma unroll
                for (int m = 0; m < k; ++m) dup |= b[m] == b[k];
                if (dup || cnt >= threshold) continue;
                const uint2 r = __ldg(ranges + b[k]);   // (~start, end); (0, 0) = empty
                for (uint32_t s = ~r.x; s < r.y && cnt < threshold; ++s) {
                    const float4 q = spos[s];
                    const float dx = __fsub_rn(q.x, p.x), dy = __fsub_rn(q.y, p.y), dz = __fsub_rn(q.z, p.z);
                    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                    cnt += d2 < r2 ? 1u : 0u;
                }
            }
        }
        sel = cnt < threshold;
        const uint32_t i = ids[t];
        const float v = sel ? 1.0f : 0.0f;
        pos_w[(size_t)i * 4] = v;
        block_w[(size_t)i * block_stride] = v;
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, sel);
    if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(selected, (uint32_t)__popc(ballot));
}

// Every visibility set to `v` (threshold 0, or a radius whose square rounds to 0: no count can matter).
__global__ void __launch_bounds__(SEL_THREADS) select_fill_kernel(uint32_t n, float v, float* __restrict__ pos_w,
                                                                  float* __restrict__ block_w, uint32_t block_stride) {
    const uint32_t i = blockIdx.x * SEL_THREADS + threadIdx.x;
    if (i >= n) return;
    pos_w[(size_t)i * 4] = v;
    block_w[(size_t)i * block_stride] = v;
}

// ---- host side -----------------------------------------------------------------------------------------------------
// Buckets of a cloud of n gaussians: a power of two >= n, at least 2^10, at most 2^24.
uint32_t select_num_buckets(uint32_t n) {
    uint32_t b = 1u << 10;
    while (b < n && b < (1u << 24)) b <<= 1;
    return b;
}
// 8-bit digit places of the sort over keys [0, n_buckets] (the sentinel included)
int select_sort_passes(uint32_t n_buckets) {
    int bits = 0;
    while ((1u << bits) <= n_buckets) ++bits;
    return (bits + 7) / 8;
}

static uint32_t sel_grid(uint32_t n) { return (n + SEL_THREADS - 1) / SEL_THREADS; }

void launch_select_keys(const float4* pos, uint32_t n, float radius, uint32_t n_buckets, uint32_t* keys, uint32_t* vals,
                        uint32_t* n_sort, cudaStream_t stream) {
    select_keys_kernel<<<sel_grid(n), SEL_THREADS, 0, stream>>>(pos, n, sel_cell_size(radius), n_buckets, keys, vals, n_sort);
}

void launch_select_count(const float4* pos, const uint32_t* ids, const uint2* ranges, uint32_t n, float radius, uint32_t n_buckets,
                         float r2, uint32_t threshold, float4* spos, float* pos_w, float* block_w, uint32_t block_stride,
                         uint32_t* selected, cudaStream_t stream) {
    select_gather_kernel<<<sel_grid(n), SEL_THREADS, 0, stream>>>(pos, ids, n, spos);
    select_count_kernel<<<sel_grid(n), SEL_THREADS, 0, stream>>>(spos, ids, ranges, n, sel_cell_size(radius), n_buckets - 1u, r2,
                                                                 threshold, pos_w, block_w, block_stride, selected);
}

void launch_select_fill(uint32_t n, float v, float* pos_w, float* block_w, uint32_t block_stride, cudaStream_t stream) {
    select_fill_kernel<<<sel_grid(n), SEL_THREADS, 0, stream>>>(n, v, pos_w, block_w, block_stride);
}

}  // namespace bgs
