// bin.cu -- stage 4: tile binning / range build (SURVEY.md §8 row a7; no counterpart in the
// reference, which rasterises one instanced quad per gaussian: src/render/mod.rs:1562-1566).
//
// For every visible splat in front-to-back rank order, emit one (tile id, rank) pair per 16x16
// tile its conservative pixel bbox touches (payload = the splat's record index).  Pair offsets are an
// exclusive scan of the per-splat tile counts in rank order, so the stable tile-id radix sort that
// follows yields, per tile, a slice of the GLOBAL depth order.
#include "common.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int BIN_THREADS = 256;
constexpr int COOP_ITEMS = 8;        // cooperative kernel: up to 8 ranks per thread per round
constexpr uint32_t BIN_TINY = 4u;   // footprints up to this many tiles: written by the owning thread
constexpr uint32_t BIN_BIG = 128u;   // larger than this: global queue, drained by the whole grid

// Cooperative variant (all CTAs co-resident).  Each CTA owns a contiguous range of front-to-back ranks.
//   phase 1: per splat, the tiles its bbox touches; the CTA publishes THREE totals: pairs, medium-footprint splats,
//            large-footprint splats (bboxes stay in registers when the range is a single sub-tile -- the usual case)
//   -- grid barrier --
//   phase 2: exclusive prefixes of the three totals over the earlier CTAs (parallel sums, no atomics, no chained
//            look-back): tiny footprints (<= 4 tiles) are written right away by the owning thread; medium ones go to the
//            front of the queue arrays, large ones to the back, each at its prefix position (rank order preserved)
//   -- grid barrier --
//   phase 3: the whole grid drains both queues, statically partitioned (warp w takes medium batches w, w + W, ...:
//            a shared head counter cost one contended atomic per warp -- 4736 of them -- just to learn the queue was empty)
__device__ __forceinline__ void block_sum_prefix3(const uint32_t* cnt3, uint32_t upto, uint64_t out[3], unsigned long long* s_red64 /*[3][8]*/) {
    uint64_t v0 = 0, v1 = 0, v2 = 0;
    for (uint32_t p = threadIdx.x; p < upto; p += BIN_THREADS) {
        v0 += ld_volatile(cnt3 + 3 * p); v1 += ld_volatile(cnt3 + 3 * p + 1); v2 += ld_volatile(cnt3 + 3 * p + 2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v0 += __shfl_xor_sync(0xffffffffu, v0, o); v1 += __shfl_xor_sync(0xffffffffu, v1, o); v2 += __shfl_xor_sync(0xffffffffu, v2, o);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) { s_red64[warp] = v0; s_red64[8 + warp] = v1; s_red64[16 + warp] = v2; }
    __syncthreads();
    out[0] = out[1] = out[2] = 0;
#pragma unroll
    for (int w = 0; w < BIN_THREADS / 32; ++w) { out[0] += s_red64[w]; out[1] += s_red64[8 + w]; out[2] += s_red64[16 + w]; }
    __syncthreads();
}

// VIEWS (bgs_render_views): a splat's tile ids are its view's, tile0[i] + ty tiles_x(i) + tx; its view is its global
// index's (slot_ids[record index] / n_view), looked up where the pairs are written: by the owning thread, and for the
// medium and large queues by the warp that drains the entry.  (A one-view frame has tile0 = 0 and tiles_x.)
template <bool VIEWS>
__device__ __forceinline__ void bin_emit_body(const SplatRec* __restrict__ recs, const uint32_t* __restrict__ perm,
                                              FrameCounters* __restrict__ ctr, ChunkCounters* __restrict__ cc, uint32_t frac_a,
                                              uint32_t frac_b, uint32_t num_tiles_total, uint32_t* __restrict__ block_cnt,
                                              int tiles_x, uint32_t capacity, uint32_t* __restrict__ pair_keys,
                                              uint32_t* __restrict__ pair_vals, uint32_t* __restrict__ q_rank,
                                              uint32_t* __restrict__ q_off, uint32_t q_cap, uint32_t* __restrict__ sticky_need,
                                              const uint32_t* __restrict__ slot_ids, const ViewTable* vt) {
    // record index r's first tile id and row length
    auto tile_base = [&](uint32_t r, uint32_t& base, uint32_t& row) {
        base = 0u; row = (uint32_t)tiles_x;
        if constexpr (VIEWS) {
            const uint32_t i = vt->view_of(__ldg(slot_ids + r));
            base = vt->tile0[i]; row = (uint32_t)vt->tiles_x[i];
        }
    };
    __shared__ uint32_t s_wtot[3][BIN_THREADS / 32];
    __shared__ unsigned long long s_red64[3 * 8];
    __shared__ uint32_t s_tot[3];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t G = gridDim.x, b = blockIdx.x;
    const uint32_t n_vis = ctr->n_vis;
    // this round's front-to-back rank range [ra, rb) = n_vis * [frac_a, frac_b) / 65536 (the whole visible set in a
    // one-round frame); empty once every tile has saturated in the earlier rounds (nothing left to blend into)
    uint32_t ra = (uint32_t)((uint64_t)n_vis * frac_a >> 16), rb = (uint32_t)((uint64_t)n_vis * frac_b >> 16);
    if (frac_a != 0u && ld_volatile(&ctr->tiles_done) >= num_tiles_total) {
        if (b == 0 && t == 0) cc->skipped = 1u;
        rb = ra;
    }
    const uint32_t n_rng = rb - ra;
    if (n_rng == 0u) return;   // (grid-uniform) nothing to emit: the round's counters stay zero
    // this CTA's contiguous rank range, cut into sub-tiles of 256 * ipt ranks (ipt chosen so that the whole
    // range is ONE sub-tile whenever it fits 8 items per thread: every CTA then does the same number of rounds)
    const uint32_t rlo = ra + (uint32_t)((uint64_t)b * n_rng / G), rhi = ra + (uint32_t)((uint64_t)(b + 1) * n_rng / G);
    const uint32_t chunk = (n_rng + G - 1) / G;
    uint32_t ipt = (chunk + BIN_THREADS - 1) / BIN_THREADS;
    if (ipt > COOP_ITEMS) ipt = COOP_ITEMS;
    if (ipt == 0) ipt = 1;
    const uint32_t sub = BIN_THREADS * ipt;
    const bool single = rhi - rlo <= sub;     // one sub-tile: phase 2 reuses phase 1's registers

    // the bboxes of this thread's ranks [r0, r0 + ipt): all rank -> record-index loads first, then all bbox loads
    // (two dependent L2 round trips for the whole batch instead of two per splat)
    uint32_t bx[COOP_ITEMS], by[COOP_ITEMS], cnt[COOP_ITEMS], ri[COOP_ITEMS];
    auto load_items = [&](uint32_t r0) {
#pragma unroll
        for (int j = 0; j < COOP_ITEMS; ++j) {
            const uint32_t r = r0 + j;
            const bool ok = (uint32_t)j < ipt && r < rhi;
            ri[j] = ok ? (perm ? __ldg(perm + (n_vis - 1u - r)) : r) : 0xFFFFFFFFu;   // rank -> record index
        }
#pragma unroll
        for (int j = 0; j < COOP_ITEMS; ++j) {
            uint2 bb = make_uint2(1u, 1u);                                             // (empty bbox: lo = 1 > hi = 0)
            if (ri[j] != 0xFFFFFFFFu) bb = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const char*>(recs + ri[j]) + 24));
            bx[j] = bb.x; by[j] = bb.y;
            const uint32_t xlo = bb.x & 0xFFFFu, xhi = bb.x >> 16, ylo = bb.y & 0xFFFFu, yhi = bb.y >> 16;
            cnt[j] = (xlo <= xhi && ylo <= yhi) ? ((xhi >> 4) - (xlo >> 4) + 1u) * ((yhi >> 4) - (ylo >> 4) + 1u) : 0u;
            if (ri[j] == 0xFFFFFFFFu) ri[j] = 0u;
        }
    };

    // ---- phase 1
    uint32_t mine = 0u, mmed = 0u, mbig = 0u;
    for (uint32_t base = rlo; base < rhi; base += sub) {
        load_items(base + t * ipt);
#pragma unroll
        for (int j = 0; j < COOP_ITEMS; ++j) {
            mine += cnt[j];
            mmed += (cnt[j] > BIN_TINY && cnt[j] <= BIN_BIG) ? 1u : 0u;
            mbig += cnt[j] > BIN_BIG ? 1u : 0u;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mine += __shfl_xor_sync(0xffffffffu, mine, o); mmed += __shfl_xor_sync(0xffffffffu, mmed, o); mbig += __shfl_xor_sync(0xffffffffu, mbig, o);
    }
    if (lane == 0) { s_wtot[0][warp] = mine; s_wtot[1][warp] = mmed; s_wtot[2][warp] = mbig; }
    __syncthreads();
    if (t < 3) {
        uint32_t tot = 0u;
#pragma unroll
        for (int w = 0; w < BIN_THREADS / 32; ++w) tot += s_wtot[t][w];
        if (t == 0 && tot > LB_VMASK) tot = LB_VMASK;
        s_tot[t] = tot;
        st_volatile(block_cnt + 3 * b + t, tot);
    }
    grid_barrier(&cc->barrier, G);

    // ---- phase 2 (pair sums saturate at 2^30 - 1: such a frame is rejected by the host)
    uint64_t pre[3];
    block_sum_prefix3(block_cnt, b, pre, s_red64);
    if (b == G - 1 && t == 0) {
        const uint64_t need64 = pre[0] + s_tot[0];
        const uint32_t need = need64 > LB_VMASK ? LB_VMASK : (uint32_t)need64;
        cc->n_pairs_needed = need;
        cc->n_pairs = need < capacity ? need : capacity;
        cc->med_count = (uint32_t)(pre[1] + s_tot[1]);
        cc->big_count = (uint32_t)(pre[2] + s_tot[2]);
        atomicMax(sticky_need, need);
        if (need > capacity) ctr->truncated = 1u;
    }
    uint32_t run = pre[0] > LB_VMASK ? LB_VMASK : (uint32_t)pre[0];
    uint32_t mrun = (uint32_t)pre[1], brun = (uint32_t)pre[2];
    for (uint32_t base = rlo; base < rhi; base += sub) {
        const uint32_t r0 = base + t * ipt;
        uint32_t tmine = 0u, nbig = 0u, nmed = 0u;
        if (!single) load_items(r0);
#pragma unroll
        for (int j = 0; j < COOP_ITEMS; ++j) {
            tmine += cnt[j];
            nbig += cnt[j] > BIN_BIG ? 1u : 0u;
            nmed += (cnt[j] > BIN_TINY && cnt[j] <= BIN_BIG) ? 1u : 0u;
        }
        uint32_t incl = tmine, bincl = nbig, mincl = nmed;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            const uint32_t z = __shfl_up_sync(0xffffffffu, bincl, o);
            const uint32_t x = __shfl_up_sync(0xffffffffu, mincl, o);
            if (lane >= o) { incl += y; bincl += z; mincl += x; }
        }
        if (lane == 31) { s_wtot[0][warp] = incl; s_wtot[1][warp] = mincl; s_wtot[2][warp] = bincl; }
        __syncthreads();
        uint32_t wprefix = 0u, ttotal = 0u, bprefix = 0u, btotal = 0u, mprefix = 0u, mtotal = 0u;
#pragma unroll
        for (int w = 0; w < BIN_THREADS / 32; ++w) {
            const uint32_t c = s_wtot[0][w], e = s_wtot[1][w], d = s_wtot[2][w];
            if (w < warp) { wprefix += c; bprefix += d; mprefix += e; }
            ttotal += c; btotal += d; mtotal += e;
        }
        // footprint classes:  <= BIN_TINY tiles: written right here by the owning thread;
        //   <= BIN_BIG: medium queue (front of the queue arrays), drained 32 splats per warp in phase 3;
        //   larger: big queue (back of the queue arrays), one splat (or a part of one) per warp in phase 3
        uint32_t off = run + wprefix + incl - tmine;
        uint32_t qat = brun + bprefix + bincl - nbig;
        uint32_t mat = mrun + mprefix + mincl - nmed;
#pragma unroll
        for (int j = 0; j < COOP_ITEMS; ++j) {
            if (cnt[j] == 0u) continue;
            if (cnt[j] > BIN_BIG) {
                q_rank[q_cap - 1u - qat] = ri[j]; q_off[q_cap - 1u - qat] = off; ++qat;
            } else if (cnt[j] > BIN_TINY) {
                q_rank[mat] = ri[j]; q_off[mat] = off; ++mat;
            } else {
                const uint32_t txlo = (bx[j] & 0xFFFFu) >> 4, txhi = (bx[j] >> 16) >> 4;
                const uint32_t tylo = (by[j] & 0xFFFFu) >> 4, tyhi = (by[j] >> 16) >> 4;
                uint32_t o = off, kb, kx;
                tile_base(ri[j], kb, kx);
                for (uint32_t ty = tylo; ty <= tyhi; ++ty)
                    for (uint32_t tx = txlo; tx <= txhi; ++tx) {
                        if (o < capacity) {
                            pair_keys[o] = kb + ty * kx + tx;
                            pair_vals[o] = ri[j];
                        }
                        ++o;
                    }
            }
            off += cnt[j];
        }
        run += ttotal; mrun += mtotal; brun += btotal;
        __syncthreads();
    }
    grid_barrier(&cc->barrier, 2u * G);

    // ---- phase 3a: medium footprints, 32 per warp: each lane fetches one splat's (record, offset, bbox)
    //      so the memory latency is paid once per 32 splats; then the warp writes them one after another
    // warp w of CTA b is global warp w * G + b: consecutive batches (the queues are in rank order, so the first ones hold
    // the nearest = largest footprints) land on different CTAs / SMs
    const uint32_t gwarp = (uint32_t)warp * G + b, total_warps = G * (BIN_THREADS / 32);
    const uint32_t nm = ld_volatile(&cc->med_count);
    for (uint32_t mb = gwarp * 32u; mb < nm; mb += total_warps * 32u) {
        const uint32_t i = mb + lane;
        uint32_t m_ri = 0u, m_off = 0u, m_txlo = 0u, m_tylo = 0u, m_w = 1u, m_total = 0u;
        if (i < nm) {
            m_ri = __ldcg(q_rank + i); m_off = __ldcg(q_off + i);
            const uint2 bb = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const char*>(recs + m_ri) + 24));
            m_txlo = (bb.x & 0xFFFFu) >> 4; m_tylo = (bb.y & 0xFFFFu) >> 4;
            m_w = ((bb.x >> 16) >> 4) - m_txlo + 1u;
            m_total = m_w * (((bb.y >> 16) >> 4) - m_tylo + 1u);
        }
        for (int sI = 0; sI < 32; ++sI) {
            const uint32_t total = __shfl_sync(0xffffffffu, m_total, sI);
            if (total == 0u) continue;
            const uint32_t r = __shfl_sync(0xffffffffu, m_ri, sI), off = __shfl_sync(0xffffffffu, m_off, sI);
            const uint32_t txlo = __shfl_sync(0xffffffffu, m_txlo, sI), tylo = __shfl_sync(0xffffffffu, m_tylo, sI);
            const uint32_t w = __shfl_sync(0xffffffffu, m_w, sI);
            uint32_t kb, kx;
            tile_base(r, kb, kx);
            for (uint32_t k = lane; k < total; k += 32) {
                const uint32_t o = off + k;
                if (o < capacity) {
                    const uint32_t qy = k / w;
                    pair_keys[o] = kb + (tylo + qy) * kx + (txlo + (k - qy * w));
                    pair_vals[o] = r;
                }
            }
        }
    }
    // ---- phase 3b: large footprints from the back queue, one (part of a) splat per warp
    //      (a few splats that each cover thousands of tiles -- the front of a heavy scene -- are cut into up to
    //      16 parts so the whole grid shares them)
    const uint32_t nq = ld_volatile(&cc->big_count);
    uint32_t part_shift = 0u;
    while (part_shift < 4u && ((uint64_t)nq << (part_shift + 2u)) <= (uint64_t)total_warps) ++part_shift;
    const uint32_t n_tickets = nq << part_shift;
    // (tickets are dealt round-robin starting at the LAST warp so the warps that drained medium batches get fewer)
    for (uint32_t tk = total_warps - 1u - gwarp; tk < n_tickets; tk += total_warps) {
        const uint32_t part = tk & ((1u << part_shift) - 1u);
        const uint32_t q = tk >> part_shift;
        const uint32_t r = __ldcg(q_rank + (q_cap - 1u - q)), off = __ldcg(q_off + (q_cap - 1u - q));
        const uint2 bb = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const char*>(recs + r) + 24));
        const uint32_t txlo = (bb.x & 0xFFFFu) >> 4, txhi = (bb.x >> 16) >> 4;
        const uint32_t tylo = (bb.y & 0xFFFFu) >> 4, tyhi = (bb.y >> 16) >> 4;
        const uint32_t w = txhi - txlo + 1u, total_all = w * (tyhi - tylo + 1u);
        // this part's slice [i0, total) of the footprint, in multiples of 32 pairs
        const uint32_t per = (((total_all + (1u << part_shift) - 1u) >> part_shift) + 31u) & ~31u;
        const uint32_t i0 = part * per;
        if (i0 >= total_all) continue;
        const uint32_t total = min(total_all, i0 + per);
        uint32_t ty = tylo + (i0 + (uint32_t)lane) / w, tx = txlo + (i0 + (uint32_t)lane) % w;
        const uint32_t dy = 32u / w, dxr = 32u % w;
        uint32_t kb, kx;
        tile_base(r, kb, kx);
        for (uint32_t i = i0 + lane; i < total; i += 32) {
            const uint32_t o = off + i;
            if (o < capacity) {
                pair_keys[o] = kb + ty * kx + tx;
                pair_vals[o] = r;
            }
            ty += dy; tx += dxr;
            if (tx > txhi) { tx -= w; ++ty; }
        }
    }
}

__global__ void __launch_bounds__(BIN_THREADS)
bin_emit_coop_kernel(const SplatRec* __restrict__ recs, const uint32_t* __restrict__ perm, FrameCounters* __restrict__ ctr,
                     ChunkCounters* __restrict__ cc, uint32_t frac_a, uint32_t frac_b, uint32_t num_tiles_total,
                     uint32_t* __restrict__ block_cnt /* [grid][3] */, int tiles_x, uint32_t capacity, uint32_t* __restrict__ pair_keys,
                     uint32_t* __restrict__ pair_vals, uint32_t* __restrict__ q_rank, uint32_t* __restrict__ q_off,
                     uint32_t q_cap, uint32_t* __restrict__ sticky_need) {
    bin_emit_body<false>(recs, perm, ctr, cc, frac_a, frac_b, num_tiles_total, block_cnt, tiles_x, capacity, pair_keys, pair_vals,
                         q_rank, q_off, q_cap, sticky_need, nullptr, nullptr);
}

// bgs_render_views' binning: one round over every view's splats, each into its own view's tiles
__global__ void __launch_bounds__(BIN_THREADS)
bin_emit_views_kernel(const SplatRec* __restrict__ recs, const uint32_t* __restrict__ perm, FrameCounters* __restrict__ ctr,
                      ChunkCounters* __restrict__ cc, uint32_t num_tiles_total, uint32_t* __restrict__ block_cnt,
                      uint32_t capacity, uint32_t* __restrict__ pair_keys, uint32_t* __restrict__ pair_vals,
                      uint32_t* __restrict__ q_rank, uint32_t* __restrict__ q_off, uint32_t q_cap,
                      uint32_t* __restrict__ sticky_need, const uint32_t* __restrict__ slot_ids,
                      const __grid_constant__ ViewTable vt) {
    bin_emit_body<true>(recs, perm, ctr, cc, 0u, 65536u, num_tiles_total, block_cnt, 0, capacity, pair_keys, pair_vals, q_rank,
                        q_off, q_cap, sticky_need, slot_ids, &vt);
}

int bin_coop_blocks_per_sm() {
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, bin_emit_coop_kernel, BIN_THREADS, 0) != cudaSuccess) return 0;
    return b;
}
cudaError_t launch_bin_emit_coop(const SplatRec* recs, const uint32_t* perm, FrameCounters* ctr, ChunkCounters* cc,
                                 uint32_t frac_a, uint32_t frac_b, uint32_t num_tiles_total, uint32_t* block_cnt,
                                 int tiles_x, uint32_t capacity, uint32_t* pair_keys, uint32_t* pair_vals,
                                 uint32_t* q_rank, uint32_t* q_off, uint32_t q_cap, uint32_t grid, uint32_t* sticky_need, cudaStream_t stream) {
    void* args[] = {(void*)&recs, (void*)&perm, (void*)&ctr, (void*)&cc, (void*)&frac_a, (void*)&frac_b, (void*)&num_tiles_total,
                    (void*)&block_cnt, (void*)&tiles_x, (void*)&capacity, (void*)&pair_keys,
                    (void*)&pair_vals, (void*)&q_rank, (void*)&q_off, (void*)&q_cap, (void*)&sticky_need};
    return cudaLaunchCooperativeKernel((const void*)bin_emit_coop_kernel, dim3(grid), dim3(BIN_THREADS), args, 0, stream);
}
cudaError_t launch_bin_emit_views(const SplatRec* recs, const uint32_t* perm, FrameCounters* ctr, ChunkCounters* cc,
                                  uint32_t num_tiles_total, uint32_t* block_cnt, uint32_t capacity, uint32_t* pair_keys,
                                  uint32_t* pair_vals, uint32_t* q_rank, uint32_t* q_off, uint32_t q_cap, uint32_t grid,
                                  uint32_t* sticky_need, const uint32_t* slot_ids, const ViewTable& vt, int sm_count,
                                  cudaStream_t stream) {
    // (the grid is planned for bin_emit_coop_kernel: no larger than this kernel's co-resident CTAs)
    static const int per_sm = [] {
        int b = 0;
        return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, bin_emit_views_kernel, BIN_THREADS, 0) == cudaSuccess ? b : 0;
    }();
    if (per_sm == 0) return cudaErrorNotSupported;
    grid = grid < (uint32_t)(per_sm * sm_count) ? grid : (uint32_t)(per_sm * sm_count);
    void* args[] = {(void*)&recs, (void*)&perm, (void*)&ctr, (void*)&cc, (void*)&num_tiles_total, (void*)&block_cnt,
                    (void*)&capacity, (void*)&pair_keys, (void*)&pair_vals, (void*)&q_rank, (void*)&q_off, (void*)&q_cap,
                    (void*)&sticky_need, (void*)&slot_ids, (void*)&vt};
    return cudaLaunchCooperativeKernel((const void*)bin_emit_views_kernel, dim3(grid), dim3(BIN_THREADS), args, 0, stream);
}

}  // namespace bgs
