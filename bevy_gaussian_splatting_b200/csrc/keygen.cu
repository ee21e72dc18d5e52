// keygen.cu -- stage 1: depth-key generation + stable stream compaction of the visible set.
//
// Replaces radix_sort_a's key half (src/sort/radix.wgsl:86-106): key = 0xFFFFFFFF - bits(|Mp-cam|^2)
// for in-frustum gaussians, 0xFFFFFFFF otherwise, shifted by 32 - depth_bits.  Instead of sorting
// the culled (all-ones) keys with everything else, the visible (key, index) pairs are compacted
// IN INDEX ORDER (keygen_coop_kernel), so the stable LSD sort that follows sees the same tie order
// as the reference; the culled tail of the reference's sorted_entry_buffer is "ascending index"
// and is reconstructed only by the debug hook.  BGS_FLAG_SORT_ALL keeps every entry (keygen_all_kernel).
//
// HBM-bound streaming kernel: 16 B read per gaussian (coalesced float4), 8 B written per
// visible gaussian.  Compiled with -fmad=false (see project_math.cuh).
#include "project_math.cuh"
#include "entry_src.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int KG_THREADS = 256;
constexpr int KG_ITEMS = 8;
constexpr int KG_TILE = KG_THREADS * KG_ITEMS;

// BGS_FLAG_SORT_ALL (reference-literal mode): every entry goes to the depth sort in index order, payload = the
// gaussian index; only the visible ones are counted
__global__ void __launch_bounds__(KG_THREADS)
keygen_all_kernel(const float4* __restrict__ pos, uint32_t n, FrameConsts fc, uint32_t* __restrict__ keys_out,
                  uint32_t* __restrict__ ids_out, FrameCounters* __restrict__ ctr) {
    const uint32_t i = blockIdx.x * KG_THREADS + threadIdx.x;
    bool vis = false;
    if (i < n) {
        float pw[4];
        keygen_world_pos(fc, __ldcs(pos + i), pw);
        vis = in_frustum_fast(fc, pw);
        keys_out[i] = depth_key(fc, vis, cam_dist2(fc, pw));
        ids_out[i] = i;
    }
    const int cnt = __syncthreads_count(vis);
    if (threadIdx.x == 0 && cnt) atomicAdd(&ctr->n_vis, (uint32_t)cnt);
    if (i == 0) ctr->n_sort = n;
}

// Cooperative variant (all CTAs co-resident, launched with cudaLaunchCooperativeKernel): each CTA owns a
// CONTIGUOUS range of 2048-gaussian tiles.
//   phase 1 streams the positions once (16 B/gaussian, the only HBM traffic that scales with N), decides
//           visibility, and keeps just ONE BIT per gaussian (warp ballots -> a 4 B mask word per 32 gaussians in an
//           L2-resident scratch) plus the CTA's visible count.  No key is computed for the ~88 % that are culled.
//   -- one grid barrier --
//   phase 2 sums the counts of all earlier CTAs in parallel, scans its own mask words, and expands them: visible
//           element e of the CTA (found by binary search over the word prefix + select-nth-bit) re-reads its position
//           (L2 / 32 B sectors, visible ones only), computes the key and writes (key, index, slot) at run + e --
//           fully coalesced, in index order, so the stable LSD sort sees the reference's tie order.
//           The depth sort's digit histograms are accumulated on the way (shared-memory atomics, visible keys only:
//           at ~2 cycles per lane-atomic they are most of this phase's time, more than the position re-read).
constexpr int KG_WORDS_PER_TILE = KG_TILE / 32;    // 64 mask words
constexpr int KG_CHUNK_WORDS = 1024;               // phase 2 expands 1024 words (32 K gaussians) at a time

// The positions come from a Src (entry_src.cuh): one cloud or a scene's segment table.  Both phases walk their indices
// upwards, so a thread finds its first index's segment once and advances from there.
template <class Src>
__device__ __forceinline__ void keygen_coop_body(const Src& src, uint32_t n, const FrameConsts& fc, uint32_t* __restrict__ masks,
                                                 uint32_t* __restrict__ keys_out, uint32_t* __restrict__ ids_out,
                                                 uint32_t* __restrict__ slots_out, uint32_t* __restrict__ block_cnt,
                                                 FrameCounters* __restrict__ ctr, uint32_t* __restrict__ hist, int hist_passes) {
    __shared__ uint32_t s_hist[4 * 256];   // digit histograms of the visible keys (the depth sort's pre-pass, fused)
    __shared__ uint32_t s_red[KG_THREADS / 32];
    __shared__ uint32_t s_total;
    __shared__ uint32_t s_mask[KG_CHUNK_WORDS];
    __shared__ uint32_t s_pref[KG_CHUNK_WORDS];   // exclusive prefix of popc(s_mask)
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t G = gridDim.x, b = blockIdx.x;
    const uint32_t tiles_total = (n + KG_TILE - 1) / KG_TILE;
    const uint32_t t0 = (uint32_t)((uint64_t)b * tiles_total / G), t1 = (uint32_t)((uint64_t)(b + 1) * tiles_total / G);

    // ---- phase 1: one visibility bit per gaussian of this CTA's range, visible count
    uint32_t mine = 0u;                      // (warp-uniform: every lane counts its warp's ballots)
    uint32_t cmin_inv = 0u, cmax_p1 = 0u;   // Depth mode only: extremes of the culled indices
    uint32_t sj = src.seg(t0 * KG_TILE + warp * (32 * KG_ITEMS) + lane);
    for (uint32_t tile = t0; tile < t1; ++tile) {
        // warp w covers 256 consecutive gaussians of the tile, item j = 32 consecutive ones (coalesced 512 B loads)
        const uint32_t wbase = tile * KG_TILE + warp * (32 * KG_ITEMS);
        float4 p[KG_ITEMS];
        const uint32_t sj0 = sj;   // (the second loop walks the segments again from here)
#pragma unroll
        for (int j = 0; j < KG_ITEMS; ++j) {
            const uint32_t i = wbase + j * 32 + lane;
            if (i < n) sj = src.advance(sj, i);
            p[j] = (i < n) ? __ldcs(src.pos_at(sj, i)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        uint32_t myword = 0u, sk = sj0;
#pragma unroll
        for (int j = 0; j < KG_ITEMS; ++j) {
            const uint32_t i = wbase + j * 32 + lane;
            bool v = false;
            if (i < n) {
                sk = src.advance(sk, i);
                float pw[4];
                keygen_world_pos(src.fc(sk), p[j], pw);
                v = in_frustum_fast(src.fc(sk), pw);
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, v);
            mine += __popc(bal);
            if (lane == j) myword = bal;
            if ((fc.rasterize_mode == BGS_RASTERIZE_DEPTH || fc.aux) && i < n && !v) { cmin_inv = max(cmin_inv, 0xFFFFFFFFu - i); cmax_p1 = max(cmax_p1, i + 1u); }
        }
        if (lane < KG_ITEMS) __stcg(masks + (size_t)tile * KG_WORDS_PER_TILE + warp * KG_ITEMS + lane, myword);
    }
    if (lane == 0) s_red[warp] = mine;
    if ((fc.rasterize_mode == BGS_RASTERIZE_DEPTH || fc.aux)) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            cmin_inv = max(cmin_inv, __shfl_xor_sync(0xffffffffu, cmin_inv, o));
            cmax_p1 = max(cmax_p1, __shfl_xor_sync(0xffffffffu, cmax_p1, o));
        }
        if (lane == 0 && cmax_p1) { atomicMax(&ctr->culled_min_inv, cmin_inv); atomicMax(&ctr->culled_max_p1, cmax_p1); }
    }
    __syncthreads();
    if (t == 0) {
        uint32_t tot = 0u;
#pragma unroll
        for (int w = 0; w < KG_THREADS / 32; ++w) tot += s_red[w];
        s_total = tot;
        st_volatile(block_cnt + b, tot);
    }
    grid_barrier(&ctr->barrier[0], G);

    // ---- phase 2: exclusive prefix over CTAs, then ordered expansion of this CTA's mask words
    for (int i = t; i < hist_passes * 256; i += KG_THREADS) s_hist[i] = 0u;
    uint32_t run = block_sum_prefix<KG_THREADS>(block_cnt, b, s_red);
    if (b == G - 1 && t == 0) { ctr->n_vis = run + s_total; ctr->n_sort = run + s_total; }
    const uint32_t w_begin = t0 * KG_WORDS_PER_TILE, w_end = t1 * KG_WORDS_PER_TILE;
    uint32_t ej = src.seg(t0 * KG_TILE);
    for (uint32_t wc = w_begin; wc < w_end; wc += KG_CHUNK_WORDS) {
        const uint32_t cw = min((uint32_t)KG_CHUNK_WORDS, w_end - wc);
        // each thread owns 4 consecutive words of the chunk: local prefix, then a block scan of the per-thread sums
        uint32_t m[4], c[4], tsum = 0u;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t w = (uint32_t)t * 4u + k;
            m[k] = (w < cw) ? __ldcg(masks + wc + w) : 0u;
            c[k] = tsum;
            tsum += __popc(m[k]);
        }
        uint32_t incl = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_red[warp] = incl;
        __syncthreads();
        uint32_t wprefix = 0u, chunk_total = 0u;
#pragma unroll
        for (int w = 0; w < KG_THREADS / 32; ++w) {
            const uint32_t v = s_red[w];
            if (w < warp) wprefix += v;
            chunk_total += v;
        }
        const uint32_t texcl = wprefix + incl - tsum;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            s_mask[t * 4 + k] = m[k];
            s_pref[t * 4 + k] = texcl + c[k];
        }
        __syncthreads();
        for (uint32_t e = t; e < chunk_total; e += KG_THREADS) {
            // largest word w with s_pref[w] <= e (words with no visible gaussian share their successor's prefix: the
            // search lands on the LAST of them or on the word itself; skip forward over empty words by construction:
            // upper_bound - 1 always holds a word whose range [pref, pref + popc) contains e)
            uint32_t lo = 0u, hi = KG_CHUNK_WORDS;             // invariant: s_pref[lo] <= e, (hi == size or s_pref[hi] > e)
#pragma unroll
            for (int it = 0; it < 10; ++it) {
                const uint32_t mid = (lo + hi) >> 1;
                if (s_pref[mid] <= e) lo = mid; else hi = mid;
            }
            const uint32_t r = e - s_pref[lo];
            const uint32_t bit = __fns(s_mask[lo], 0u, (int)r + 1);
            const uint32_t i = (wc + lo) * 32u + bit;
            ej = src.advance(ej, i);
            const FrameConsts& fi = src.fc(ej);
            float pw[4];
            keygen_world_pos(fi, __ldg(src.pos_at(ej, i)), pw);
            const uint32_t key = depth_key(fi, true, cam_dist2(fi, pw));
            const uint32_t dst = run + e;
            keys_out[dst] = key;
            ids_out[dst] = i;          // compact slot -> gaussian index
            slots_out[dst] = dst;      // the sort's payload: the compact slot
            for (int pp = 0; pp < hist_passes; ++pp) atomicAdd(&s_hist[pp * 256 + ((key >> (8 * pp)) & 255u)], 1u);
        }
        run += chunk_total;
        __syncthreads();
    }
    for (int i = t; i < hist_passes * 256; i += KG_THREADS) {
        const uint32_t c = s_hist[i];
        if (c) atomicAdd(&hist[i], c);
    }
}

__global__ void __launch_bounds__(KG_THREADS)
keygen_coop_kernel(const float4* __restrict__ pos, uint32_t n, FrameConsts fc, uint32_t* __restrict__ masks,
                   uint32_t* __restrict__ keys_out, uint32_t* __restrict__ ids_out, uint32_t* __restrict__ slots_out,
                   uint32_t* __restrict__ block_cnt, FrameCounters* __restrict__ ctr, uint32_t* __restrict__ hist,
                   int hist_passes) {
    keygen_coop_body(OneCloud{pos, fc}, n, fc, masks, keys_out, ids_out, slots_out, block_cnt, ctr, hist, hist_passes);
}

// bgs_render_scene: the same over the N global indices of a segment table (ids_out holds global indices).  fc of
// segment 0 carries the frame-wide values.
__global__ void __launch_bounds__(KG_THREADS)
keygen_scene_kernel(SceneTable tab, uint32_t* __restrict__ masks, uint32_t* __restrict__ keys_out,
                    uint32_t* __restrict__ ids_out, uint32_t* __restrict__ slots_out, uint32_t* __restrict__ block_cnt,
                    FrameCounters* __restrict__ ctr, uint32_t* __restrict__ hist, int hist_passes) {
    keygen_coop_body(SceneSrc{tab}, tab.n_total, tab.seg[0].fc, masks, keys_out, ids_out, slots_out, block_cnt, ctr, hist,
                     hist_passes);
}

// bgs_render_entities_many: the same over a segment table in device memory.  fc carries the frame-wide values (its
// rasterize_mode and aux), as segment 0's do for keygen_scene_kernel.
__global__ void __launch_bounds__(KG_THREADS)
keygen_many_kernel(SceneTableDev tab, FrameConsts fc, uint32_t* __restrict__ masks, uint32_t* __restrict__ keys_out,
                   uint32_t* __restrict__ ids_out, uint32_t* __restrict__ slots_out, uint32_t* __restrict__ block_cnt,
                   FrameCounters* __restrict__ ctr, uint32_t* __restrict__ hist, int hist_passes) {
    keygen_coop_body(SceneSrcDev{tab}, tab.n_total, fc, masks, keys_out, ids_out, slots_out, block_cnt, ctr, hist, hist_passes);
}

// Debug hook: rebuild the reference's full sorted_entry_buffer (sort/mod.rs:323-329) from the
// compacted result: [0, n_vis) = sorted visible entries, then every culled index ascending
// with key 0xFFFFFFFF >> shift.  Single block per call chunk; not on the hot path.
template <class Src>
__device__ __forceinline__ void culled_flags_body(const Src& src, uint32_t n, uint32_t* __restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t j = src.seg(i);
    const FrameConsts& fc = src.fc(j);
    const float4 p = *src.pos_at(j, i);
    float pw[4], ndc[2];
    mat4_point(fc.model, p.x, p.y, p.z, pw);
    flags[i] = in_frustum(fc, pw, ndc) ? 0u : 1u;
}

__global__ void culled_flags_kernel(const float4* __restrict__ pos, uint32_t n, FrameConsts fc,
                                    uint32_t* __restrict__ flags) {
    culled_flags_body(OneCloud{pos, fc}, n, flags);
}

__global__ void culled_flags_scene_kernel(SceneTable tab, uint32_t* __restrict__ flags) {
    culled_flags_body(SceneSrc{tab}, tab.n_total, flags);
}

__global__ void culled_flags_many_kernel(SceneTableDev tab, uint32_t* __restrict__ flags) {
    culled_flags_body(SceneSrcDev{tab}, tab.n_total, flags);
}

void launch_keygen_all(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* keys_out, uint32_t* ids_out,
                       FrameCounters* ctr, cudaStream_t stream) {
    keygen_all_kernel<<<(n + KG_THREADS - 1) / KG_THREADS, KG_THREADS, 0, stream>>>(pos, n, fc, keys_out, ids_out, ctr);
}

int keygen_coop_blocks_per_sm() {
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, keygen_coop_kernel, KG_THREADS, 0) != cudaSuccess) return 0;
    return b;
}
cudaError_t launch_keygen_coop(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* masks, uint32_t* keys_out,
                               uint32_t* ids_out, uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr,
                               uint32_t* hist, int hist_passes, uint32_t grid, cudaStream_t stream) {
    FrameConsts fcc = fc;
    void* args[] = {(void*)&pos, (void*)&n, (void*)&fcc, (void*)&masks, (void*)&keys_out, (void*)&ids_out,
                    (void*)&slots_out, (void*)&block_cnt, (void*)&ctr, (void*)&hist, (void*)&hist_passes};
    return cudaLaunchCooperativeKernel((const void*)keygen_coop_kernel, dim3(grid), dim3(KG_THREADS), args, 0, stream);
}

void launch_culled_flags(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* flags, cudaStream_t stream) {
    culled_flags_kernel<<<(n + 255) / 256, 256, 0, stream>>>(pos, n, fc, flags);
}

int keygen_scene_blocks_per_sm() {
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, keygen_scene_kernel, KG_THREADS, 0) != cudaSuccess) return 0;
    return b;
}
cudaError_t launch_keygen_scene(const SceneTable& tab, uint32_t* masks, uint32_t* keys_out, uint32_t* ids_out,
                                uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr, uint32_t* hist, int hist_passes,
                                uint32_t grid, cudaStream_t stream) {
    void* args[] = {(void*)&tab, (void*)&masks, (void*)&keys_out, (void*)&ids_out, (void*)&slots_out, (void*)&block_cnt,
                    (void*)&ctr, (void*)&hist, (void*)&hist_passes};
    return cudaLaunchCooperativeKernel((const void*)keygen_scene_kernel, dim3(grid), dim3(KG_THREADS), args, 0, stream);
}

void launch_culled_flags_scene(const SceneTable& tab, uint32_t* flags, cudaStream_t stream) {
    culled_flags_scene_kernel<<<(tab.n_total + 255) / 256, 256, 0, stream>>>(tab, flags);
}

int keygen_many_blocks_per_sm() {
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, keygen_many_kernel, KG_THREADS, 0) != cudaSuccess) return 0;
    return b;
}
cudaError_t launch_keygen_many(const SceneTableDev& tab, const FrameConsts& fc, uint32_t* masks, uint32_t* keys_out,
                               uint32_t* ids_out, uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr, uint32_t* hist,
                               int hist_passes, uint32_t grid, cudaStream_t stream) {
    SceneTableDev t = tab;
    FrameConsts f = fc;
    void* args[] = {(void*)&t, (void*)&f, (void*)&masks, (void*)&keys_out, (void*)&ids_out, (void*)&slots_out,
                    (void*)&block_cnt, (void*)&ctr, (void*)&hist, (void*)&hist_passes};
    return cudaLaunchCooperativeKernel((const void*)keygen_many_kernel, dim3(grid), dim3(KG_THREADS), args, 0, stream);
}

void launch_culled_flags_many(const SceneTableDev& tab, uint32_t* flags, cudaStream_t stream) {
    culled_flags_many_kernel<<<(tab.n_total + 255) / 256, 256, 0, stream>>>(tab, flags);
}

}  // namespace bgs
