// radix.cu -- stage 2 (and the tile-id sort of stage 4): stable LSD radix sort, 8-bit digits, ALL digit
// places of one sort inside ONE cooperative launch.
//
// Replaces radix_sort_b / radix_sort_c_count_tiles / radix_sort_c_scan_tiles / radix_sort_c_scatter
// (src/sort/radix.wgsl:110-279) and the 3P+3 dispatches of run_radix_sort (src/sort/radix.rs:672-754).  Same
// contract: ascending by key, stable (ties keep input order), P = depth_bits / 8 passes
// (src/render/mod.rs:715-745).  The entry count comes from device memory (n_ptr): no host round-trip sits
// between key-gen and the sort.
//
// Each pass is a "onesweep": a CTA loads a tile, ranks it per warp (stable), publishes the tile's digit counts,
// obtains its global digit offsets by decoupled look-back over the predecessors' counts, and scatters.  The
// passes of a sort are separated by a grid barrier instead of a kernel boundary (the keys/payload of a depth
// sort at C3 are 5.8 MB: they never leave L2), tiles are assigned statically (tile = blockIdx.x + k * grid:
// all CTAs are co-resident, predecessors are always in flight), and the look-back status words carry a
// per-launch epoch so they never need clearing.
//   optional phase 0: the digit histograms of all passes (pair sort; the depth sort gets them from key-gen)
//   optional epilogue of the last pass: per-tile ranges of the sorted pair list (a7) -- replaces a separate
//   pass over the sorted keys.
//
// HBM/L2-bound: per pass 8 B read + 8 B written per entry; histogram phase reads 4 B per entry.
#include "common.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int RS_THREADS = 512;                   // fat CTAs, one (two beyond 8 K entries x SMs) per SM: a single-wave sort has
constexpr int RS_WARPS = RS_THREADS / 32;         // <= one (two) tiles per SM, so the look-back walks (traffic ~ tiles^2 x 2 KB)
                                                  // stay short; 512 x 64 registers leave half an SM to a concurrent kernel
constexpr int RS_TABLE_WORDS = RS_WARPS * 256;    // one peer-mask table (all warps)
constexpr int RS_MIN_CTAS = 2;                    // two co-resident CTAs per SM: caps the kernel at 64 registers
constexpr int LB_BATCH = 16;                      // look-back loads in flight per thread

// status word: [63:34] epoch, [33:32] flag (1 = tile aggregate, 2 = inclusive prefix), [31:0] value
constexpr unsigned long long ST_AGG = 1ull << 32, ST_INC = 2ull << 32;
__device__ __forceinline__ unsigned long long ld_status(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_status(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

struct SortParams {
    uint32_t* keys[2];
    uint32_t* vals[2];
    const uint32_t* n_ptr;          // entries to sort (device)
    uint32_t* hist;                 // [passes][256] raw digit counts (zero on entry when compute_hist)
    unsigned long long* status;     // [passes][status_stride] look-back words
    size_t status_stride;           // words per pass = max tiles * 256
    uint32_t epoch;                 // unique per launch within the status array's lifetime, never 0
    uint32_t* barrier;              // grid barrier word, zero on entry
    int passes;
    int shift0;                     // pass p sorts on bits [shift0 + 8p, shift0 + 8p + 8)
    int compute_hist;
    uint2* ranges;                  // non-null: the keys are tile ids; the last pass emits ranges[id] = (~start, end)
};

constexpr size_t radix_smem_bytes(int items) {
    const size_t tile = (size_t)RS_THREADS * items;
    const size_t kv = tile > (size_t)RS_TABLE_WORDS ? tile : (size_t)RS_TABLE_WORDS;
    return (2 * kv + (size_t)RS_WARPS * 256 + 256 + 256 + 1024 + RS_WARPS) * 4;
}

template <int RS_ITEMS, bool MASK_TABLE>
__global__ void __launch_bounds__(RS_THREADS, RS_MIN_CTAS)
radix_coop_kernel(SortParams P) {
    constexpr int RS_TILE = RS_THREADS * RS_ITEMS;
    constexpr int KV_WORDS = RS_TILE > RS_TABLE_WORDS ? RS_TILE : RS_TABLE_WORDS;
    extern __shared__ __align__(16) uint32_t s_dyn[];
    uint32_t* s_keys = s_dyn;                                   // [KV_WORDS]  (first: peer-mask table B)
    uint32_t* s_vals = s_keys + KV_WORDS;                       // [KV_WORDS]  (first: peer-mask table A)
    uint32_t (*s_whist)[256] = reinterpret_cast<uint32_t (*)[256]>(s_vals + KV_WORDS);   // per-warp digit counts -> offsets
    uint32_t* s_binstart = &s_whist[0][0] + RS_WARPS * 256;     // [256] tile-local exclusive digit offsets
    uint32_t* s_gbase = s_binstart + 256;                       // [256] global destination of digit d's run, minus s_binstart[d]
    uint32_t* s_wtot = s_gbase + 256 + 1024;                    // [RS_WARPS] (the 1024 words between: look-back window sums / flags)

    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t G = gridDim.x;
    const uint32_t n = *P.n_ptr;
    const uint32_t num_tiles = (n + RS_TILE - 1) / RS_TILE;
    uint32_t bar_target = 0u;

    // ---- phase 0 (optional): digit histograms of every pass in one read of the keys
    if (P.compute_hist) {
        uint32_t* s_hist = &s_whist[0][0];        // [passes <= 4][256]
        for (int i = t; i < P.passes * 256; i += RS_THREADS) s_hist[i] = 0u;
        __syncthreads();
        const uint32_t* kin = P.keys[0];
        for (uint32_t base = blockIdx.x * RS_TILE; base < n; base += G * RS_TILE) {
            uint32_t k[RS_ITEMS];
#pragma unroll
            for (int j = 0; j < RS_ITEMS; ++j) {
                const uint32_t i = base + j * RS_THREADS + t;
                k[j] = (i < n) ? __ldcg(kin + i) : 0u;
            }
            for (int p = 0; p < P.passes; ++p) {
                // a thread's consecutive keys often share a digit (clustered tile ids / depth keys): merge runs
                uint32_t run_d = 0xFFFFFFFFu, run_c = 0u;
#pragma unroll
                for (int j = 0; j < RS_ITEMS; ++j) {
                    const uint32_t i = base + j * RS_THREADS + t;
                    if (i >= n) break;
                    const uint32_t d = (k[j] >> (P.shift0 + 8 * p)) & 255u;
                    if (d == run_d) { ++run_c; }
                    else {
                        if (run_c) atomicAdd(&s_hist[p * 256 + run_d], run_c);
                        run_d = d; run_c = 1u;
                    }
                }
                if (run_c) atomicAdd(&s_hist[p * 256 + run_d], run_c);
            }
        }
        __syncthreads();
        for (int i = t; i < P.passes * 256; i += RS_THREADS) {
            const uint32_t c = s_hist[i];
            if (c) atomicAdd(&P.hist[i], c);
        }
        bar_target += G;
        grid_barrier(P.barrier, bar_target);
    }

    const unsigned long long ep = (unsigned long long)P.epoch << 34;
    int cur = 0;
    for (int p = 0; p < P.passes; ++p, cur ^= 1) {
        const int shift = P.shift0 + 8 * p;
        // (selects, not P.keys[cur]: a dynamically indexed kernel parameter would be copied to local memory)
        const uint32_t* __restrict__ keys_in = cur ? P.keys[1] : P.keys[0];
        const uint32_t* __restrict__ vals_in = cur ? P.vals[1] : P.vals[0];
        uint32_t* __restrict__ keys_out = cur ? P.keys[0] : P.keys[1];
        uint32_t* __restrict__ vals_out = cur ? P.vals[0] : P.vals[1];
        unsigned long long* status = P.status + (size_t)p * P.status_stride;
        const bool emit_ranges = P.ranges != nullptr && p == P.passes - 1;

        for (uint32_t tile = blockIdx.x; tile < num_tiles; tile += G) {
            const uint32_t tile_base = tile * RS_TILE;
            // warp-striped load: warp w owns [w*32*ITEMS, (w+1)*32*ITEMS) of the tile; item j = 32 consecutive entries
            uint32_t k[RS_ITEMS];
            const uint32_t my_base = tile_base + warp * (32 * RS_ITEMS) + lane;
#pragma unroll
            for (int j = 0; j < RS_ITEMS; ++j) {
                const uint32_t i = my_base + j * 32;
                k[j] = (i < n) ? __ldcg(keys_in + i) : 0xFFFFFFFFu;   // padding sorts to the tile's tail
            }
            // (thread t clears column t & 255 of 8 of the 32 per-warp rows; ditto the two peer-mask tables)
#pragma unroll
            for (int i = 0; i < RS_WARPS * 256 / RS_THREADS; ++i) (&s_whist[0][0])[i * RS_THREADS + t] = 0u;
            if (MASK_TABLE) {
#pragma unroll
                for (int i = 0; i < RS_TABLE_WORDS / RS_THREADS; ++i) { s_vals[i * RS_THREADS + t] = 0u; s_keys[i * RS_THREADS + t] = 0u; }
            }
            __syncthreads();

            // stable in-warp ranking: entries of one digit are ranked in (item, lane) order
            uint32_t rank[RS_ITEMS];
#pragma unroll
            for (int j = 0; j < RS_ITEMS; ++j) {
                const uint32_t d = (k[j] >> shift) & 255u;
                uint32_t peers, old;
                if (MASK_TABLE) {
                    // small (latency-bound) sorts: peers via a per-warp mask table in shared memory (the tables alias
                    // s_vals / s_keys, unused until the scatter; even / odd items alternate tables so the clear of one
                    // item never races the next item's ORs): one ATOMS.OR per lane, conflicts only among lanes sharing
                    // the digit.  Cheaper than MATCH.ANY when the sort is latency-bound.
                    uint32_t* mm = ((j & 1) ? s_keys : s_vals) + warp * 256;
                    atomicOr(&mm[d], 1u << lane);
                    __syncwarp();
                    peers = mm[d];
                    old = s_whist[warp][d];               // every lane reads the running count itself (broadcast)
                    __syncwarp();
                    if (lane == 31 - __clz(peers)) { mm[d] = 0u; s_whist[warp][d] = old + __popc(peers); }
                } else {
                    // large (throughput-bound) sorts: MATCH.ANY (the mask table's atomics cost more there than they save)
                    peers = __match_any_sync(0xffffffffu, d);
                    old = s_whist[warp][d];
                    __syncwarp();
                    if (lane == 31 - __clz(peers)) s_whist[warp][d] = old + __popc(peers);
                    __syncwarp();
                }
                rank[j] = old + __popc(peers & lanemask_lt());
            }
            __syncthreads();

            const uint32_t tile_end = tile_base + RS_TILE;
            const uint32_t pad = (tile_end > n) ? (tile_end - n) : 0u;
            // threads 0..255 own one digit each: exclusive scan across warps, tile totals, look-back
            uint32_t cnt = 0u, cnt_valid = 0u, incl = 0u, gh = 0u, gh_incl = 0u;
            unsigned long long* my_status = status + (size_t)tile * 256 + (t & 255);
            if (t < 256) {
#pragma unroll 8
                for (int w = 0; w < RS_WARPS; ++w) {
                    const uint32_t c = s_whist[w][t];
                    s_whist[w][t] = cnt;
                    cnt += c;
                }
                cnt_valid = (t == 255) ? cnt - pad : cnt;   // padding is all digit 255
                if (tile != 0) st_status(my_status, ep | ST_AGG | cnt_valid);   // published as early as possible
                // tile-local exclusive scan over digits (padding included: it defines smem positions)
                incl = cnt;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += y;
                }
                // tile 0 seeds the chain with the exclusive scan of the global histogram
                if (tile == 0) {
                    gh = __ldcg(P.hist + p * 256 + t);
                    gh_incl = gh;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t y = __shfl_up_sync(0xffffffffu, gh_incl, o);
                        if (lane >= o) gh_incl += y;
                    }
                }
                if (lane == 31) { s_wtot[warp] = incl; s_wtot[8 + warp] = gh_incl; }
            }
            __syncthreads();
            uint32_t binstart = 0u, excl = 0u;
            if (t < 256) {
                uint32_t wprefix = 0u, gp = 0u;
                for (int w = 0; w < warp; ++w) { wprefix += s_wtot[w]; gp += s_wtot[8 + w]; }
                binstart = wprefix + incl - cnt;
                s_binstart[t] = binstart;
                if (tile == 0) {
                    excl = gp + gh_incl - gh;
                    st_status(my_status, ep | ST_INC | (excl + cnt_valid));
                }
            }
            __syncthreads();

            // scatter into tile-sorted order in shared memory (the predecessors' words arrive meanwhile; the mask
            // tables aliasing s_keys / s_vals were last touched before the two barriers above)
#pragma unroll
            for (int j = 0; j < RS_ITEMS; ++j) {
                const uint32_t d = (k[j] >> shift) & 255u;
                const uint32_t i = my_base + j * 32;
                const uint32_t pos = rank[j] + s_binstart[d] + s_whist[warp][d];
                s_keys[pos] = k[j];
                s_vals[pos] = (i < n) ? __ldcg(vals_in + i) : 0u;
            }

            // decoupled look-back: digit d = t & 255 is walked by TWO threads (halves h = t >> 8) that take alternate
            // 16-tile windows of predecessors; the windows of a round are combined in distance order through shared
            // memory.  In a single-wave sort every tile publishes its aggregate at about the same time and nobody but
            // tile 0 holds an inclusive prefix yet, so a tile walks all the way back: two windows per round halve that
            // latency.
            if (tile != 0) {
                uint32_t* s_part = s_binstart + 512;            // [2][256] window sums (after s_binstart, s_gbase)
                uint32_t* s_fnd = s_part + 512;                 // [2][256] window ended at an inclusive prefix
                const int d = t & 255, h = t >> 8;
                const unsigned long long* ps = status + (size_t)tile * 256 + d;
                bool done = false;
                for (uint32_t round = 0;; ++round) {
                    const uint32_t w0 = (2u * round + (uint32_t)h) * LB_BATCH;   // this half's window: distances w0 + 1 .. w0 + 16
                    uint32_t sum = 0u;
                    bool found = false;
                    if (!done) {
                        unsigned long long w[LB_BATCH];
#pragma unroll
                        for (int q = 0; q < LB_BATCH; ++q)
                            w[q] = (w0 + (uint32_t)q < tile) ? ld_status(ps - (size_t)256 * (w0 + q + 1)) : (ep | ST_INC);   // (before tile 0: prefix 0)
#pragma unroll
                        for (int q = 0; q < LB_BATCH; ++q) {
                            if (!found) {
                                unsigned long long x = w[q];
                                while ((x >> 34) != (ep >> 34) || ((x >> 32) & 3ull) == 0ull) x = ld_status(ps - (size_t)256 * (w0 + q + 1));
                                sum += (uint32_t)x;
                                found = ((x >> 32) & 3ull) == 2ull;
                            }
                        }
                    }
                    s_part[h * 256 + d] = sum;
                    s_fnd[h * 256 + d] = found ? 1u : 0u;
                    __syncthreads();
                    if (!done) {
                        excl += s_part[d];
                        if (s_fnd[d]) done = true;
                        else { excl += s_part[256 + d]; done = s_fnd[256 + d] != 0u; }
                    }
                    if (__syncthreads_and(done ? 1 : 0)) break;     // (also fences the reuse of s_part / s_fnd)
                }
                if (t < 256) st_status(my_status, ep | ST_INC | (excl + cnt_valid));
            }
            if (t < 256) s_gbase[t] = excl - binstart;
            __syncthreads();

            // coalesced write-out: consecutive positions of one digit land on consecutive addresses
            const uint32_t valid = RS_TILE - pad;
#pragma unroll 4
            for (uint32_t q = t; q < valid; q += RS_THREADS) {
                const uint32_t kk = s_keys[q];
                const uint32_t dst = s_gbase[(kk >> shift) & 255u] + q;
                keys_out[dst] = kk;
                vals_out[dst] = s_vals[q];
                if (emit_ranges) {
                    // equal tile ids are contiguous in the tile (the input is sorted by the lower digits, the ranking is
                    // stable) and in the output: each run's first / last element records the slice bounds
                    if (q == 0u || s_keys[q - 1] != kk) atomicMax(&P.ranges[kk].x, ~dst);
                    if (q == valid - 1u || s_keys[q + 1] != kk) atomicMax(&P.ranges[kk].y, dst + 1u);
                }
            }
            __syncthreads();
        }
        if (p + 1 < P.passes) {
            bar_target += G;
            grid_barrier(P.barrier, bar_target);
        }
    }
}

// ---- host-side launch helpers ------------------------------------------------------------------
// look-back status rows (tiles per pass) a sort of up to `capacity` entries may need: launch_radix_sort never picks
// a tile smaller than capacity / rows entries
uint32_t radix_num_tiles(uint32_t capacity) {
    const uint32_t need = capacity / (RS_THREADS * 16u) + 1u;
    return need > 4096u ? need : 4096u;
}

namespace {
template <int ITEMS, bool MASK>
cudaError_t radix_launch_variant(const SortParams& P, uint32_t grid, cudaStream_t stream) {
    static bool attr_set[64] = {};   // per device (the opt-in shared-memory size is a per-device function attribute)
    const size_t smem = radix_smem_bytes(ITEMS);
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(radix_coop_kernel<ITEMS, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
    SortParams p = P;
    void* args[] = {(void*)&p};
    return cudaLaunchCooperativeKernel((const void*)radix_coop_kernel<ITEMS, MASK>, dim3(grid), dim3(RS_THREADS), args, smem, stream);
}
}  // namespace

// co-resident CTAs per SM of the largest variant (2 expected: 82 KB of shared memory, 64 registers x 512 threads)
int radix_coop_blocks_per_sm(int) {
    int b = 0;
    if (cudaFuncSetAttribute(radix_coop_kernel<16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)radix_smem_bytes(16)) != cudaSuccess) return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, radix_coop_kernel<16, false>, RS_THREADS, radix_smem_bytes(16)) != cudaSuccess) return 0;
    return b;
}

// One stable LSD sort of *n_ptr (key, payload) entries on bits [shift0, shift0 + 8 * passes).  The result lands in
// keys[passes & 1] / vals[passes & 1].  n_hint (expected entry count, e.g. last frame's) only picks the tile size and
// the grid -- one wave of sm_count (or 2 x sm_count) fat CTAs covers the sort whenever the count allows; correctness
// never depends on it.  `coop_per_sm` = radix_coop_blocks_per_sm().
cudaError_t launch_radix_sort(uint32_t* keys0, uint32_t* vals0, uint32_t* keys1, uint32_t* vals1, const uint32_t* n_ptr,
                              uint32_t capacity, uint32_t n_hint, uint32_t* hist, int compute_hist, void* status,
                              size_t status_stride, uint32_t epoch, uint32_t* barrier, int passes, int shift0, uint2* ranges,
                              int sm_count, int coop_per_sm, cudaStream_t stream) {
    SortParams P;
    P.keys[0] = keys0; P.keys[1] = keys1; P.vals[0] = vals0; P.vals[1] = vals1;
    P.n_ptr = n_ptr; P.hist = hist; P.status = reinterpret_cast<unsigned long long*>(status); P.status_stride = status_stride;
    P.epoch = epoch; P.barrier = barrier; P.passes = passes; P.shift0 = shift0; P.compute_hist = compute_hist;
    P.ranges = ranges;
    if (n_hint > capacity) n_hint = capacity;
    // items per thread so that `waves` waves of tiles cover the expected count with ~3 % head-room (a frame that outgrows
    // it gives some CTAs one more tile: slower, never wrong).  One CTA per SM when the count allows, else two -- unless
    // the caller caps it (coop_per_sm = 1: queued frames keep the sort's footprint at half an SM and run two waves).
    const uint64_t want = (uint64_t)n_hint + n_hint / 32 + 1024;
    uint32_t grid = (uint32_t)sm_count;
    auto items_for = [&](uint32_t g, uint32_t& waves) {
        const uint64_t per_wave = (uint64_t)g * RS_THREADS * 16u;
        waves = (uint32_t)((want + per_wave - 1) / per_wave);
        const uint64_t per_item = (uint64_t)g * RS_THREADS * waves;
        return (uint32_t)((want + per_item - 1) / per_item);
    };
    uint32_t waves = 1;
    uint32_t items = items_for(grid, waves);
    if (waves > 1 && coop_per_sm >= 2) {
        grid = 2u * (uint32_t)sm_count;
        items = items_for(grid, waves);
    }
    if (waves > 3) items = 17;      // many waves: the throughput variant (16 items, MATCH.ANY ranking)
    // never more tiles than status rows, whatever the actual count turns out to be
    const uint32_t rows = (uint32_t)(status_stride / 256);
    const uint32_t min_items = (uint32_t)(((uint64_t)capacity + (uint64_t)rows * RS_THREADS - 1) / ((uint64_t)rows * RS_THREADS));
    if (items < min_items) items = min_items;
    if (items <= 2) return radix_launch_variant<2, true>(P, grid, stream);
    if (items <= 4) return radix_launch_variant<4, true>(P, grid, stream);
    if (items <= 6) return radix_launch_variant<6, true>(P, grid, stream);
    if (items <= 8) return radix_launch_variant<8, true>(P, grid, stream);
    if (items <= 10) return radix_launch_variant<10, true>(P, grid, stream);
    if (items <= 12) return radix_launch_variant<12, true>(P, grid, stream);
    if (items <= 16) return radix_launch_variant<16, true>(P, grid, stream);
    return radix_launch_variant<16, false>(P, grid, stream);   // multi-wave (throughput-bound) sorts: MATCH.ANY ranking
}

}  // namespace bgs
