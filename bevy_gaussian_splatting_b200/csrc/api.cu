// api.cu -- the extern "C" boundary of libbgs (include/bgs.h): contexts, clouds, the per-view
// frame (stage orchestration on one CUDA stream), parity/debug hooks, stage timing.
//
// No PyTorch, no wgpu, no CPU fallback: every stage is a hand-written sm_90a kernel.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <mutex>
#include <new>
#include <vector>

#include "common.cuh"

namespace bgs {
// keygen.cu
void launch_keygen_all(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* keys_out, uint32_t* ids_out,
                       FrameCounters* ctr, cudaStream_t stream);
int keygen_coop_blocks_per_sm();
cudaError_t launch_keygen_coop(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* masks, uint32_t* keys_out,
                               uint32_t* ids_out, uint32_t* slots_out, uint32_t* block_cnt, FrameCounters* ctr,
                               uint32_t* hist, int hist_passes, uint32_t grid, cudaStream_t stream);
void launch_culled_flags(const float4* pos, uint32_t n, const FrameConsts& fc, uint32_t* flags, cudaStream_t stream);
// radix.cu
uint32_t radix_num_tiles(uint32_t capacity);
int radix_coop_blocks_per_sm(int items);
cudaError_t launch_radix_sort(uint32_t* keys0, uint32_t* vals0, uint32_t* keys1, uint32_t* vals1, const uint32_t* n_ptr,
                              uint32_t capacity, uint32_t n_hint, uint32_t* hist, int compute_hist, void* status,
                              size_t status_stride, uint32_t epoch, uint32_t* barrier, int passes, int shift0, uint2* ranges,
                              int sm_count, int coop_per_sm, cudaStream_t stream);
// project.cu
void launch_depth_range(const float4* pos, uint32_t n, const uint32_t* sorted_payload, const uint32_t* slot_ids,
                        FrameCounters* ctr, const FrameConsts& fc, cudaStream_t stream);
void launch_repack(bool f16, const void* pos, const void* sh, const void* rot, const void* so, uint32_t n, void* blocks,
                   cudaStream_t stream);
void launch_project(bool f16, const void* blocks, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                    const FrameConsts& fc, SplatRec* recs, float4* extra, uint32_t n_hint, int sm_count,
                    const float* cutoff_tab, float4* aux, cudaStream_t stream);
void launch_cutoff_table(float* tab, cudaStream_t stream);
// bin.cu
int bin_coop_blocks_per_sm();
cudaError_t launch_bin_emit_coop(const SplatRec* recs, const uint32_t* perm, FrameCounters* ctr, ChunkCounters* cc,
                                 uint32_t frac_a, uint32_t frac_b, uint32_t num_tiles_total, uint32_t* block_cnt,
                                 int tiles_x, uint32_t capacity, uint32_t* pair_keys, uint32_t* pair_vals,
                                 uint32_t* q_rank, uint32_t* q_off, uint32_t q_cap, uint32_t grid,
                                 uint32_t* sticky_need, cudaStream_t stream);
// raster.cu
void launch_raster(int mode, bool large_footprints, const SplatRec* recs, const float4* extra, const uint32_t* tile_entries,
                   const uint2* ranges, int W, int H, int tiles_x, int tiles_y, void* out, uint32_t format,
                   const float4* aux, void* out_depth, void* out_normal, cudaStream_t stream);
void launch_raster_round(const SplatRec* recs, const uint32_t* tile_entries, const uint2* ranges, int W, int H, int tiles_x,
                         int tiles_y, void* out, uint32_t format, float4* state, unsigned char* tile_done,
                         uint32_t* tiles_done, int first, int last, cudaStream_t stream);
}  // namespace bgs

using namespace bgs;

struct bgs_cloud {
    bgs_context* ctx;       // owning context; nulled when that context is destroyed first
    int device;             // the CUDA device the planes live on
    uint32_t n;
    bool f16;
    bool cov;         // f16 layout whose second plane holds Covariance3dOpacityPacked128 records (precomputed Sigma3D)
    float4* pos;      // n * 16 B
    void* blocks;     // gaussian-major copy of every plane (f16: n * 128 B, f32: n * 256 B), what the projection gathers
};

struct bgs_context {
    int device = 0;
    int sm_count = 132;
    uint32_t kg_grid = 0, bin_grid = 0;   // co-resident grid sizes of the cooperative kernels (synchronous frames: latency)
    uint32_t kg_grid_async = 0, bin_grid_async = 0;   // ... of queued (BGS_FLAG_ASYNC) frames: 1 CTA per SM.  A latency-bound
                                          // cooperative grid holds its registers while it waits; with several frames in flight
                                          // a smaller grid leaves that room to the other frames' issue-bound blend
    int rs_per_sm = 0;                    // co-resident radix-sort CTAs per SM (radix.cu)
    uint32_t sort_epoch = 0;              // look-back status epoch: +1 per sort launch (status words never need clearing)
    cudaStream_t stream = nullptr;    // render stream (high priority): everything but the projection
    cudaStream_t stream2 = nullptr;   // projection runs here, beside the depth sort
    cudaStream_t stream_r = nullptr;  // LOW priority: the tile blend of one-round frames.  With several contexts in flight the
                                      // latency-bound front of the next frame (high priority, cooperative grids) takes SMs as
                                      // the previous frame's short-lived raster CTAs retire, instead of queueing behind them
    cudaEvent_t ev_front = nullptr, ev_rdone = nullptr;
    cudaEvent_t ev[6] = {};
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_p0 = nullptr, ev_p1 = nullptr;
    uint32_t n_vis_hint = 0;          // last frame's visible count (sizes the projection grid)
    uint32_t n_pairs_hint = 0;        // last frame's pair count (picks the pair sort's tile size); on chunked
                                      // frames an ESTIMATE of what one round would have emitted
    uint32_t chunk_pairs_hint[MAX_CHUNKS] = {};   // last chunked frame's pairs per round (pair sort tile size)
    bool chunk_hint_valid = false;
    float4* state = nullptr;          // per-pixel blend state between rounds (tile-major), tiles * 256 * 16 B
    uint32_t cap_state_tiles = 0;
    unsigned char* tile_done = nullptr;   // in the arena (cleared per frame)
    int pend_chunks = 1, last_chunks = 1;
    char err[512] = {0};

    // scratch sized by the cloud (grow-only)
    uint32_t cap_n = 0;
    uint32_t* keys[2] = {nullptr, nullptr};
    uint32_t* vals[2] = {nullptr, nullptr};
    uint32_t* slot_ids = nullptr;     // compact slot -> gaussian index (key-gen output, index order)
    SplatRec* recs = nullptr;
    float4* extra = nullptr;          // 4 x float4 per record: 2DGS + USE_AABB only (allocated on first use)
    uint32_t cap_extra = 0;
    float4* aux = nullptr;            // 2 x float4 per record: depth / normal colour sources (bgs_render_aux only)
    uint32_t cap_aux = 0;
    void* frame_aux[2] = {nullptr, nullptr};   // depth / normal frames when bgs_render_aux delivers to host memory
    size_t frame_aux_bytes = 0;
    // scratch sized by the pair capacity (grow-only)
    uint32_t cap_pairs = 0;
    uint32_t* pkeys[2] = {nullptr, nullptr};
    uint32_t* pvals[2] = {nullptr, nullptr};
    // zeroed-per-frame arena: counters | hist | keygen CTA counts | bin CTA counts | ranges | done bytes
    uint8_t* arena = nullptr;
    size_t arena_bytes = 0;
    uint32_t arena_tiles = 0;
    // look-back status rows of the two sorts (64-bit epoch-tagged words, cleared once at allocation)
    void* status_depth = nullptr;      // [4][tiles(n)][256]
    void* status_pairs = nullptr;      // [4][tiles(cap_pairs)][256]
    uint32_t status_n = 0, status_np = 0;
    bool async_pending = false;        // a BGS_FLAG_ASYNC frame has been enqueued and not yet completed
    const bgs_cloud* pend_cloud = nullptr; uint32_t pend_n = 0; FrameConsts pend_fc; bool pend_sort_all = false, pend_by_slot = false;
    int pend_tiles_x = 0, pend_tiles_y = 0, pend_W = 0, pend_H = 0; const void* pend_target = nullptr;
    cudaEvent_t ev_done = nullptr;
    FrameCounters* ctr = nullptr;
    uint32_t* hist = nullptr;          // [8 + 4 * MAX_CHUNKS][256]: depth passes 0..3, pair passes 4..7 (round 0), 8 + 4r.. (round r)
    uint32_t* kg_block_cnt = nullptr;  // [kg_grid]: keygen_coop's per-CTA visible counts
    uint32_t* bin_block_cnt = nullptr; // [bin_grid][3]: bin_emit_coop's per-CTA pair / medium / large counts
    uint2* ranges = nullptr;           // per tile (~start, end) into the sorted pair list (0, 0 = empty)
    // frame
    void* frame = nullptr;            // frames[0]
    void* frame_alt = nullptr;        // frames[1]: async frames delivered to host memory alternate targets so
    size_t frame_bytes = 0;           //            frame k's D2H copy (copy stream) overlaps frame k+1's kernels
    int frame_toggle = 0;
    cudaStream_t stream_copy = nullptr;
    cudaEvent_t ev_raster[2] = {nullptr, nullptr}, ev_copied[2] = {nullptr, nullptr};
    bool copy_pending[2] = {false, false};
    const void* last_frame = nullptr;
    FrameCounters* h_ctr = nullptr;    // pinned
    // largest n_pairs_needed of ANY frame since the last bgs_sync / synchronous render (device word outside the
    // per-frame arena + its pinned copy): a queued async frame that overflowed the pair buffer is never missed
    float* cutoff_tab = nullptr;       // adaptive cutoff of every f16 opacity value (project.cu)
    uint32_t* d_sticky = nullptr;
    uint32_t* h_sticky = nullptr;
    std::vector<bgs_cloud*> clouds;    // clouds uploaded through this context (their ctx is nulled on destroy)

    // last-frame facts (for the debug hooks)
    bool have_frame = false;
    const bgs_cloud* last_cloud = nullptr;
    FrameConsts last_fc;
    bool last_sort_all = false;
    bool last_by_slot = false;        // records indexed by compact slot (else by front-to-back rank)
    int depth_result = 0, pair_result = 0;   // which ping-pong buffer holds the sorted result
    bgs_frame_stats stats = {};
    float stage_us[6] = {0, 0, 0, 0, 0, 0};
    bool stage_valid = false;
    uint32_t launches = 0;
};

namespace {

// live contexts: clouds may be shared by the contexts of one GPU, so destroying a cloud must clear every
// context's references to it, and destroying a context must not leave its clouds with a dangling owner
std::mutex g_registry_mu;
std::vector<bgs_context*> g_contexts;

bgs_status fail(bgs_context* ctx, bgs_status st, const char* fmt, ...) {
    if (ctx) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
        va_end(ap);
    }
    return st;
}

#define CU(ctx, call)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess)                                                                          \
            return fail(ctx, e_ == cudaErrorMemoryAllocation ? BGS_ENOMEM : BGS_ECUDA, "%s: %s", #call, \
                        cudaGetErrorString(e_));                                                        \
    } while (0)

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

constexpr uint32_t CHUNK_MAX_TILES = 65536;
// chunked frames (saturation-aware binning): the visible set is binned / sorted / blended in front-to-back rank rounds
// [CHUNK_FRAC[r], CHUNK_FRAC[r + 1]) / 65536; once every tile has saturated the remaining rounds emit nothing
// (x8 schedule: the front of a heavy scene saturates the frame within a few hundred splats)
constexpr uint32_t CHUNK_FRAC[MAX_CHUNKS + 1] = {0, 16, 128, 1024, 8192, 65536};
// CTAs per SM of the cooperative key-gen and binning grids: synchronous frames (latency), queued (BGS_FLAG_ASYNC) frames
constexpr int COOP_CTAS_PER_SM = 4, COOP_CTAS_PER_SM_ASYNC = 1;
// radix-sort CTAs per SM the pair sort of queued frames may use (1: half an SM, two waves)
constexpr int SORT_CTAS_PER_SM_ASYNC = 1;

int pair_passes(uint32_t num_tiles) {
    int bits = 1;
    while ((1u << bits) < num_tiles) ++bits;
    return (bits + 7) / 8;
}

bgs_status ensure_cloud_scratch(bgs_context* c, uint32_t n) {
    if (n <= c->cap_n) return BGS_OK;
    for (int i = 0; i < 2; ++i) {
        cudaFree(c->keys[i]); cudaFree(c->vals[i]);
        c->keys[i] = c->vals[i] = nullptr;
    }
    cudaFree(c->recs); c->recs = nullptr;
    cudaFree(c->slot_ids); c->slot_ids = nullptr;
    c->cap_n = 0;
    for (int i = 0; i < 2; ++i) {
        // (>= 1024 words: keys[1] doubles as key-gen's visibility-mask scratch, one word per 32 gaussians rounded up to a tile)
        CU(c, cudaMalloc(&c->keys[i], (size_t)(n < 1024u ? 1024u : n) * 4));
        CU(c, cudaMalloc(&c->vals[i], (size_t)(n < 1024u ? 1024u : n) * 4));
    }
    CU(c, cudaMalloc(&c->slot_ids, (size_t)n * 4));
    CU(c, cudaMalloc(&c->recs, (size_t)n * sizeof(SplatRec)));
    c->cap_n = n;
    return BGS_OK;
}

bgs_status ensure_pair_scratch(bgs_context* c, uint32_t pairs) {
    if (pairs <= c->cap_pairs) return BGS_OK;
    for (int i = 0; i < 2; ++i) {
        cudaFree(c->pkeys[i]); cudaFree(c->pvals[i]);
        c->pkeys[i] = c->pvals[i] = nullptr;
    }
    c->cap_pairs = 0;
    for (int i = 0; i < 2; ++i) {
        // +64 words: the raster's 16 B-granular bulk copies may read a few entries past the last pair
        CU(c, cudaMalloc(&c->pkeys[i], ((size_t)pairs + 64) * 4));
        CU(c, cudaMalloc(&c->pvals[i], ((size_t)pairs + 64) * 4));
    }
    c->cap_pairs = pairs;
    return BGS_OK;
}

bgs_status ensure_arena(bgs_context* c, uint32_t tiles) {
    if (c->arena && tiles <= c->arena_tiles) return BGS_OK;
    tiles = tiles > c->arena_tiles ? tiles : c->arena_tiles;
    cudaFree(c->arena); c->arena = nullptr;
    size_t off = 0;
    const size_t o_ctr = off; off = align_up(off + sizeof(FrameCounters), 256);
    const size_t o_hist = off; off = align_up(off + (8 + 4 * MAX_CHUNKS) * 256 * 4, 256);
    // (the queued-frame grids are never larger than the synchronous ones)
    const size_t o_kgc = off; off = align_up(off + (size_t)c->kg_grid * 4, 256);
    const size_t o_binc = off; off = align_up(off + (size_t)c->bin_grid * 3 * 4, 256);
    // chunked frames (only for <= CHUNK_MAX_TILES tiles) use one ranges array per round + a done byte per tile; an
    // arena sized by a larger frame must still hold them for a later, smaller (chunkable) frame
    const size_t chunk_tiles = tiles <= CHUNK_MAX_TILES ? tiles : CHUNK_MAX_TILES;
    const size_t range_entries = chunk_tiles * MAX_CHUNKS > tiles ? chunk_tiles * MAX_CHUNKS : tiles;
    const size_t o_rng = off; off = align_up(off + range_entries * 8, 256);
    const size_t o_done = off; off = align_up(off + chunk_tiles, 256);
    CU(c, cudaMalloc(&c->arena, off));
    c->arena_bytes = off;
    c->ctr = reinterpret_cast<FrameCounters*>(c->arena + o_ctr);
    c->hist = reinterpret_cast<uint32_t*>(c->arena + o_hist);
    c->kg_block_cnt = reinterpret_cast<uint32_t*>(c->arena + o_kgc);
    c->bin_block_cnt = reinterpret_cast<uint32_t*>(c->arena + o_binc);
    c->ranges = reinterpret_cast<uint2*>(c->arena + o_rng);
    c->tile_done = c->arena + o_done;
    c->arena_tiles = tiles;
    return BGS_OK;
}

// look-back status rows of the sorts: 4 passes x tiles x 256 digits x 8 B, epoch-tagged (radix.cu), so they are
// cleared exactly once -- here -- and never again
bgs_status ensure_status(bgs_context* c, uint32_t n, uint32_t pairs) {
    if (n > c->status_n) {
        cudaFree(c->status_depth); c->status_depth = nullptr; c->status_n = 0;
        const size_t bytes = (size_t)4 * radix_num_tiles(n) * 256 * 8;
        CU(c, cudaMalloc(&c->status_depth, bytes));
        CU(c, cudaMemsetAsync(c->status_depth, 0, bytes, c->stream));
        c->status_n = n;
    }
    if (pairs > c->status_np) {
        cudaFree(c->status_pairs); c->status_pairs = nullptr; c->status_np = 0;
        const size_t bytes = (size_t)4 * radix_num_tiles(pairs) * 256 * 8;
        CU(c, cudaMalloc(&c->status_pairs, bytes));
        CU(c, cudaMemsetAsync(c->status_pairs, 0, bytes, c->stream));
        c->status_np = pairs;
    }
    return BGS_OK;
}

uint32_t next_epoch(bgs_context* c) {
    if (++c->sort_epoch >= (1u << 30)) {     // (2^30 sorts later) start over from clean rows
        if (c->status_depth) cudaMemsetAsync(c->status_depth, 0, (size_t)4 * radix_num_tiles(c->status_n) * 256 * 8, c->stream);
        if (c->status_pairs) cudaMemsetAsync(c->status_pairs, 0, (size_t)4 * radix_num_tiles(c->status_np) * 256 * 8, c->stream);
        c->sort_epoch = 1;
    }
    return c->sort_epoch;
}

bgs_status ensure_frame(bgs_context* c, size_t bytes) {
    if (bytes <= c->frame_bytes) return BGS_OK;
    cudaFree(c->frame); cudaFree(c->frame_alt); c->frame = c->frame_alt = nullptr; c->frame_bytes = 0;
    CU(c, cudaMalloc(&c->frame, bytes));
    CU(c, cudaMalloc(&c->frame_alt, bytes));
    CU(c, cudaMemsetAsync(c->frame, 0, bytes, c->stream));       // (BGS_FLAG_BLEND_OVER_TARGET reads the target)
    CU(c, cudaMemsetAsync(c->frame_alt, 0, bytes, c->stream));
    c->frame_bytes = bytes;
    c->copy_pending[0] = c->copy_pending[1] = false;
    return BGS_OK;
}

size_t format_bpp(uint32_t f) { return f == BGS_FORMAT_RGBA32F ? 16 : (f == BGS_FORMAT_RGBA16F ? 8 : 4); }

}  // namespace

extern "C" {

bgs_status bgs_context_create(int cuda_device, bgs_context** out) {
    if (!out) return BGS_EINVAL;
    *out = nullptr;
    bgs_context* c = new (std::nothrow) bgs_context();
    if (!c) return BGS_ENOMEM;
    c->device = cuda_device;
    cudaError_t e = cudaSetDevice(cuda_device);
    int prio_lo = 0, prio_hi = 0;
    if (e == cudaSuccess) e = cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_hi);
    if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&c->stream2, cudaStreamNonBlocking, (prio_lo + prio_hi) / 2);
    if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&c->stream_r, cudaStreamNonBlocking, prio_lo);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_front, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_rdone, cudaEventDisableTiming);
    for (int i = 0; i < 6 && e == cudaSuccess; ++i) e = cudaEventCreate(&c->ev[i]);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->stream_copy, cudaStreamNonBlocking);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
        e = cudaEventCreateWithFlags(&c->ev_raster[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventCreate(&c->ev_p0);
    if (e == cudaSuccess) e = cudaEventCreate(&c->ev_p1);
    if (e == cudaSuccess) e = cudaMallocHost(&c->h_ctr, sizeof(FrameCounters));
    if (e == cudaSuccess) e = cudaMallocHost(&c->h_sticky, 16);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_sticky, 16);
    if (e == cudaSuccess) e = cudaMemset(c->d_sticky, 0, 16);
    if (e == cudaSuccess) e = cudaMalloc(&c->cutoff_tab, 65536 * sizeof(float));
    if (e == cudaSuccess) { launch_cutoff_table(c->cutoff_tab, c->stream); e = cudaStreamSynchronize(c->stream); }
    if (e == cudaSuccess) memset(c->h_sticky, 0, 16);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, cuda_device);
    int coop = 0;   // device supports cooperative launch
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, cuda_device);
    if (e == cudaSuccess && coop) {
        const int kb = keygen_coop_blocks_per_sm(), bb = bin_coop_blocks_per_sm();
        c->kg_grid = (uint32_t)(c->sm_count * std::min(kb, COOP_CTAS_PER_SM));
        c->bin_grid = (uint32_t)(c->sm_count * std::min(bb, COOP_CTAS_PER_SM));
        c->kg_grid_async = (uint32_t)(c->sm_count * std::min(kb, COOP_CTAS_PER_SM_ASYNC));
        c->bin_grid_async = (uint32_t)(c->sm_count * std::min(bb, COOP_CTAS_PER_SM_ASYNC));
        c->rs_per_sm = radix_coop_blocks_per_sm(16);
        if (c->kg_grid == 0 || c->bin_grid == 0 || c->rs_per_sm == 0) coop = 0;
    }
    if (e == cudaSuccess && !coop) {
        snprintf(c->err, sizeof(c->err), "device %d cannot co-schedule the cooperative kernels (an sm_90a GPU such as the H100 is required)", cuda_device);
        fprintf(stderr, "libbgs: %s\n", c->err);
        e = cudaErrorNotSupported;
    }
    if (e != cudaSuccess) {
        // no CUDA device / driver: the product has no CPU path
        fprintf(stderr, "libbgs: CUDA initialisation failed on device %d: %s\n", cuda_device, cudaGetErrorString(e));
        bgs_context_destroy(c);
        return BGS_ECUDA;
    }
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);
        g_contexts.push_back(c);
    }
    *out = c;
    return BGS_OK;
}

void bgs_context_destroy(bgs_context* c) {
    if (!c) return;
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);
        g_contexts.erase(std::remove(g_contexts.begin(), g_contexts.end(), c), g_contexts.end());
        for (bgs_cloud* cl : c->clouds) cl->ctx = nullptr;   // the clouds outlive the context (destroyed by their owner later)
        c->clouds.clear();
    }
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->stream2) cudaStreamSynchronize(c->stream2);
    if (c->stream_r) { cudaStreamSynchronize(c->stream_r); cudaStreamDestroy(c->stream_r); }
    if (c->ev_front) cudaEventDestroy(c->ev_front);
    if (c->ev_rdone) cudaEventDestroy(c->ev_rdone);
    if (c->stream_copy) { cudaStreamSynchronize(c->stream_copy); cudaStreamDestroy(c->stream_copy); }
    for (int i = 0; i < 2; ++i) { if (c->ev_raster[i]) cudaEventDestroy(c->ev_raster[i]); if (c->ev_copied[i]) cudaEventDestroy(c->ev_copied[i]); }
    cudaFree(c->frame_alt);
    for (int i = 0; i < 2; ++i) {
        cudaFree(c->keys[i]); cudaFree(c->vals[i]); cudaFree(c->pkeys[i]); cudaFree(c->pvals[i]);
    }
    cudaFree(c->state);
    cudaFree(c->aux); cudaFree(c->frame_aux[0]); cudaFree(c->frame_aux[1]);
    cudaFree(c->recs); cudaFree(c->extra); cudaFree(c->slot_ids); cudaFree(c->arena); cudaFree(c->frame);
    if (c->h_ctr) cudaFreeHost(c->h_ctr);
    if (c->h_sticky) cudaFreeHost(c->h_sticky);
    cudaFree(c->d_sticky);
    cudaFree(c->cutoff_tab);
    for (int i = 0; i < 6; ++i) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
    for (cudaEvent_t e : {c->ev_fork, c->ev_join, c->ev_p0, c->ev_p1, c->ev_done}) if (e) cudaEventDestroy(e);
    cudaFree(c->status_depth); cudaFree(c->status_pairs);
    if (c->stream) cudaStreamDestroy(c->stream);
    if (c->stream2) cudaStreamDestroy(c->stream2);
    delete c;
}

static bgs_status upload_common(bgs_context* ctx, uint32_t n, bool f16, const float* pos_vis, const void* sh,
                                const void* rot, const void* so, bgs_cloud** out) {
    if (!ctx || !out) return BGS_EINVAL;
    *out = nullptr;
    if (!pos_vis || !sh || !rot || (!f16 && !so)) return fail(ctx, BGS_EINVAL, "cloud upload: null plane pointer");
    if (n == 0 || n >= (1u << 30)) return fail(ctx, BGS_EINVAL, "cloud upload: n must be in [1, 2^30)");
    CU(ctx, cudaSetDevice(ctx->device));
    bgs_cloud* cl = new (std::nothrow) bgs_cloud();
    if (!cl) return BGS_ENOMEM;
    cl->ctx = ctx; cl->device = ctx->device; cl->n = n; cl->f16 = f16; cl->cov = false;
    cl->pos = nullptr; cl->blocks = nullptr;
    // the other planes go to device scratch, are repacked into the gaussian-major blocks the projection gathers, and
    // are freed again
    void* d_sh = nullptr; void* d_rot = nullptr; void* d_so = nullptr;
    const size_t sh_bytes = (size_t)n * (f16 ? 96 : 192);
    cudaError_t e = cudaMalloc(&cl->pos, (size_t)n * 16);
    if (e == cudaSuccess) e = cudaMalloc(&d_sh, sh_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&d_rot, (size_t)n * 16);
    if (e == cudaSuccess && !f16) e = cudaMalloc(&d_so, (size_t)n * 16);
    if (e == cudaSuccess) e = cudaMemcpyAsync(cl->pos, pos_vis, (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_sh, sh, sh_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_rot, rot, (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && !f16) e = cudaMemcpyAsync(d_so, so, (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMalloc(&cl->blocks, (size_t)n * (f16 ? 128 : 256));
    if (e == cudaSuccess) {
        launch_repack(f16, cl->pos, d_sh, d_rot, d_so, n, cl->blocks, ctx->stream);
        e = cudaStreamSynchronize(ctx->stream);
    }
    cudaFree(d_sh); cudaFree(d_rot); cudaFree(d_so);
    if (e != cudaSuccess) {
        bgs_cloud_destroy(cl);
        return fail(ctx, e == cudaErrorMemoryAllocation ? BGS_ENOMEM : BGS_ECUDA, "cloud upload: %s", cudaGetErrorString(e));
    }
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);
        ctx->clouds.push_back(cl);
    }
    *out = cl;
    return BGS_OK;
}

bgs_status bgs_cloud_upload_f32(bgs_context* ctx, uint32_t n, const float* pos_vis, const float* sh,
                                const float* rot_wxyz, const float* scale_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, false, pos_vis, sh, rot_wxyz, scale_opacity, out);
}

bgs_status bgs_cloud_upload_f16(bgs_context* ctx, uint32_t n, const float* pos_vis, const uint32_t* sh_packed,
                                const uint32_t* rot_scale_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, true, pos_vis, sh_packed, rot_scale_opacity, nullptr, out);
}

bgs_status bgs_cloud_upload_f16_cov(bgs_context* ctx, uint32_t n, const float* pos_vis, const uint32_t* sh_packed,
                                    const uint32_t* cov3d_opacity, bgs_cloud** out) {
    const bgs_status s = upload_common(ctx, n, true, pos_vis, sh_packed, cov3d_opacity, nullptr, out);
    if (s == BGS_OK) (*out)->cov = true;
    return s;
}

void bgs_cloud_destroy(bgs_cloud* cl) {
    if (!cl) return;
    cudaSetDevice(cl->device);
    {
        // every live context (clouds are shared by the contexts of one GPU) drops its references: queued frames
        // that still read the planes are drained first, the debug hooks lose their frame
        std::lock_guard<std::mutex> lk(g_registry_mu);
        for (bgs_context* c : g_contexts) {
            if (c->pend_cloud == cl || c->last_cloud == cl) {
                if (c->async_pending || c->pend_cloud == cl) {
                    cudaStreamSynchronize(c->stream);
                    cudaStreamSynchronize(c->stream2);
                    cudaStreamSynchronize(c->stream_r);
                    cudaStreamSynchronize(c->stream_copy);
                }
                if (c->pend_cloud == cl) { c->pend_cloud = nullptr; c->pend_n = 0; }
                if (c->last_cloud == cl) { c->last_cloud = nullptr; c->have_frame = false; }
            }
            c->clouds.erase(std::remove(c->clouds.begin(), c->clouds.end(), cl), c->clouds.end());
        }
    }
    cudaFree(cl->pos); cudaFree(cl->blocks);
    delete cl;
}

// Bookkeeping once a frame's counters are back on the host (sync render, or bgs_sync after async ones).
static bgs_status finish_frame(bgs_context* c) {
    const int chunks = c->pend_chunks;
    uint32_t needed = 0;
    uint64_t emitted = 0;
    for (int r = 0; r < chunks; ++r) {
        const ChunkCounters& cc = c->h_ctr->chunk[r];
        needed = cc.n_pairs_needed > needed ? cc.n_pairs_needed : needed;
        emitted += cc.n_pairs;
    }
    if (needed > c->cap_pairs) {
        // the pair list (of one round) did not fit: grow (x1.25 head-room); the caller redoes the frame
        uint64_t want = (uint64_t)needed + needed / 4 + 1024;
        if (want >= (1ull << 30)) want = (1ull << 30) - 1;
        if (needed >= LB_VMASK || want <= c->cap_pairs)
            return fail(c, BGS_ENOMEM, "render: frame needs >= 2^30 (splat, tile) pairs");
        bgs_status s = ensure_pair_scratch(c, (uint32_t)want);
        if (s != BGS_OK) return s;
        return BGS_NOT_READY;
    }
    const uint32_t n = c->pend_n;   // (snapshot: the cloud may have been destroyed since the frame was queued)
    c->stage_valid = false;
    c->stats.n = n; c->stats.n_visible = c->h_ctr->n_vis; c->stats.n_pairs = emitted;
    c->stats.rounds = (uint32_t)chunks; c->stats.tiles_saturated = c->h_ctr->tiles_done;
    c->stats.tiles_x = (uint32_t)c->pend_tiles_x; c->stats.tiles_y = (uint32_t)c->pend_tiles_y;
    c->stats.width = (uint32_t)c->pend_W; c->stats.height = (uint32_t)c->pend_H;
    c->have_frame = true; c->last_cloud = c->pend_cloud; c->last_fc = c->pend_fc; c->last_sort_all = c->pend_sort_all;
    c->last_by_slot = c->pend_by_slot; c->n_vis_hint = c->h_ctr->n_vis; c->last_chunks = chunks;
    if (chunks > 1) {
        // the rounds emitted in full, scaled up to the whole visible set (the nearest splats have the largest
        // footprints, so this errs towards staying chunked)
        uint64_t got = 0;
        int full = 0;
        while (full < chunks && !c->h_ctr->chunk[full].skipped) got += c->h_ctr->chunk[full++].n_pairs_needed;
        const uint64_t est = got * 65536ull / CHUNK_FRAC[full];
        c->n_pairs_hint = est > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)est;
        for (int r = 0; r < chunks; ++r) c->chunk_pairs_hint[r] = c->h_ctr->chunk[r].n_pairs;
        c->chunk_hint_valid = true;
    } else {
        c->n_pairs_hint = c->h_ctr->chunk[0].n_pairs;
        c->chunk_hint_valid = false;
    }
    c->last_frame = c->pend_target;
    c->err[0] = 0;
    return BGS_OK;
}

bgs_status bgs_sync(bgs_context* c) {
    if (!c) return BGS_EINVAL;
    if (!c->async_pending) return BGS_OK;
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaStreamSynchronize(c->stream_copy));
    c->copy_pending[0] = c->copy_pending[1] = false;
    CU(c, cudaGetLastError());
    c->async_pending = false;
    // the sticky maximum covers EVERY frame queued since the last sync, not just the last one (whose counters are
    // in h_ctr): any of them that needed more pairs than the buffer holds was blended from a truncated list
    const uint32_t worst = c->h_sticky[0];
    const bool earlier_overflow = worst > c->cap_pairs;
    c->h_sticky[0] = 0;
    CU(c, cudaMemsetAsync(c->d_sticky, 0, 4, c->stream));
    const bgs_status s = finish_frame(c);
    if (s == BGS_NOT_READY) return fail(c, BGS_NOT_READY, "an async frame outgrew the pair buffer (now grown): render the frames queued since the last bgs_sync again");
    if (s == BGS_OK && earlier_overflow) {
        uint64_t want = (uint64_t)worst + worst / 4 + 1024;
        if (want >= (1ull << 30)) want = (1ull << 30) - 1;
        if (worst >= LB_VMASK || want <= c->cap_pairs) return fail(c, BGS_ENOMEM, "render: frame needs >= 2^30 (splat, tile) pairs");
        const bgs_status gs = ensure_pair_scratch(c, (uint32_t)want);
        if (gs != BGS_OK) return gs;
        c->have_frame = false;
        return fail(c, BGS_NOT_READY, "an earlier async frame (not the last one) outgrew the pair buffer (now grown): every frame queued since the last bgs_sync may be truncated, render them again");
    }
    return s;
}

static bgs_status render_impl(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                              const bgs_settings* st, void* out_rgba, uint32_t out_format, int out_is_device_ptr,
                              bool want_aux, void* out_depth, void* out_normal);

bgs_status bgs_render(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                      const bgs_settings* st, void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    return render_impl(c, cloud, view, uni, st, out_rgba, out_format, out_is_device_ptr, false, nullptr, nullptr);
}

bgs_status bgs_render_aux(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                          const bgs_settings* st, void* out_rgba, void* out_depth, void* out_normal, uint32_t out_format,
                          int out_is_device_ptr) {
    if (c && (!out_rgba || !out_depth || !out_normal)) return fail(c, BGS_EINVAL, "render_aux: the three output frames are required");
    if (c && st && (st->flags & BGS_FLAG_ASYNC)) return fail(c, BGS_EINVAL, "render_aux: BGS_FLAG_ASYNC is not supported");
    return render_impl(c, cloud, view, uni, st, out_rgba, out_format, out_is_device_ptr, true, out_depth, out_normal);
}

static bgs_status render_impl(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                              const bgs_settings* st, void* out_rgba, uint32_t out_format, int out_is_device_ptr,
                              bool want_aux, void* out_depth, void* out_normal) {
    if (!c) return BGS_EINVAL;
    // not-ready inputs map to the reference's silent skip-frame (radix.rs:645-658, mod.rs:1533-1539)
    if (!cloud || !view || !uni || !st) return fail(c, BGS_NOT_READY, "render: cloud/view/uniform/settings not ready");
    if (cloud->device != c->device)     // (cloud->ctx may be gone: clouds outlive the context that uploaded them)
        return fail(c, BGS_EINVAL, "render: cloud lives on another device");   // contexts of one GPU may share clouds
    if (out_format > BGS_FORMAT_RGBA32F) return fail(c, BGS_EINVAL, "render: unknown out_format %u", out_format);
    if (st->radix_sort_depth_bits != 16 && st->radix_sort_depth_bits != 24 && st->radix_sort_depth_bits != 32)
        return fail(c, BGS_EINVAL, "render: radix_sort_depth_bits must be 16, 24 or 32");
    if (st->gaussian_mode != BGS_GAUSSIAN_3D && st->gaussian_mode != BGS_GAUSSIAN_2D)
        return fail(c, BGS_EINVAL, "render: gaussian_mode %u not supported (Gaussian4d is out of scope)", st->gaussian_mode);
    if (st->rasterize_mode > BGS_RASTERIZE_POSITION)
        return fail(c, BGS_EINVAL, "render: rasterize_mode %u not supported (Color, Depth, Normal, Position are)", st->rasterize_mode);
    if (st->draw_mode > BGS_DRAW_HIGHLIGHT_SELECTED) return fail(c, BGS_EINVAL, "render: bad draw_mode");
    if (cloud->cov && (st->gaussian_mode != BGS_GAUSSIAN_3D || st->rasterize_mode == BGS_RASTERIZE_NORMAL || want_aux))
        return fail(c, BGS_EINVAL, "render: a precomputed-covariance cloud has no rotation / scale: Gaussian3d with Color, Depth or Position only");
    const int W = (int)view->viewport[2], H = (int)view->viewport[3];
    if (W <= 0 || H <= 0 || W > 65535 || H > 65535) return fail(c, BGS_EINVAL, "render: viewport %dx%d out of range", W, H);
    CU(c, cudaSetDevice(c->device));
    if (c->async_pending && !(st->flags & BGS_FLAG_ASYNC)) {
        // a synchronous render after queued frames completes them first; their failure (including an overflowed
        // pair list = BGS_NOT_READY) is the caller's to see, so this frame is not rendered on top of it
        const bgs_status ps = bgs_sync(c);
        if (ps != BGS_OK) return ps;
    }

    const uint32_t n = cloud->n;
    const int tiles_x = (W + TILE_PX - 1) / TILE_PX, tiles_y = (H + TILE_PX - 1) / TILE_PX;
    const uint32_t num_tiles = (uint32_t)tiles_x * (uint32_t)tiles_y;
    const int depth_passes = (int)st->radix_sort_depth_bits / 8;
    const int tile_passes = pair_passes(num_tiles);
    const bool sort_all = (st->flags & BGS_FLAG_SORT_ALL) != 0;

    FrameConsts fc;
    memcpy(fc.model, uni->transform, 64);
    memcpy(fc.view_from_world, view->view_from_world, 64);
    memcpy(fc.clip_from_world, view->clip_from_world, 64);
    memcpy(fc.cam, view->world_position, 12);
    fc.W = view->viewport[2]; fc.H = view->viewport[3];
    fc.p00 = view->clip_from_view[0]; fc.p11 = view->clip_from_view[5];
    fc.global_opacity = uni->global_opacity; fc.global_scale = uni->global_scale;
    fc.color_space = uni->color_space;
    fc.key_shift = 32u - st->radix_sort_depth_bits;
    fc.gaussian_mode = st->gaussian_mode; fc.rasterize_mode = st->rasterize_mode; fc.aabb = st->aabb;
    fc.adaptive = st->opacity_adaptive_radius; fc.draw_mode = st->draw_mode;
    fc.Wi = W; fc.Hi = H; fc.tiles_x = tiles_x; fc.tiles_y = tiles_y;
    fc.n_cloud = n;
    fc.aux = want_aux ? 1u : 0u;
    fc.cov_pre = cloud->cov ? 1u : 0u;
    memcpy(fc.aabb_min, uni->aabb_min, 12); memcpy(fc.aabb_max, uni->aabb_max, 12);
    static const float kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    fc.model_identity = memcmp(uni->transform, kIdentity, 64) == 0 ? 1u : 0u;   // (-0.0 entries take the general path)

    bgs_status s = ensure_cloud_scratch(c, n);
    if (s != BGS_OK) return s;
    // raster variant: 0 = quad-uv falloff (USE_OBB, 3DGS and 2DGS), 1 = 3DGS conic (USE_AABB), 2 = 2DGS ray-splat (USE_AABB)
    const int raster_mode = !st->aabb ? 0 : (st->gaussian_mode == BGS_GAUSSIAN_3D ? 1 : 2);
    if (raster_mode == 2 && c->cap_extra < c->cap_n) {
        cudaFree(c->extra); c->extra = nullptr; c->cap_extra = 0;
        CU(c, cudaMalloc(&c->extra, (size_t)c->cap_n * 64));
        c->cap_extra = c->cap_n;
    }
    void* tgt_depth = nullptr; void* tgt_normal = nullptr;
    if (want_aux) {
        if (c->cap_aux < c->cap_n) {
            cudaFree(c->aux); c->aux = nullptr; c->cap_aux = 0;
            CU(c, cudaMalloc(&c->aux, (size_t)c->cap_n * 32));
            c->cap_aux = c->cap_n;
        }
        if (out_is_device_ptr) { tgt_depth = out_depth; tgt_normal = out_normal; }
        else {
            const size_t fb = (size_t)W * H * format_bpp(out_format);
            if (fb > c->frame_aux_bytes) {
                cudaFree(c->frame_aux[0]); cudaFree(c->frame_aux[1]); c->frame_aux[0] = c->frame_aux[1] = nullptr; c->frame_aux_bytes = 0;
                CU(c, cudaMalloc(&c->frame_aux[0], fb));
                CU(c, cudaMalloc(&c->frame_aux[1], fb));
                CU(c, cudaMemsetAsync(c->frame_aux[0], 0, fb, c->stream));
                CU(c, cudaMemsetAsync(c->frame_aux[1], 0, fb, c->stream));
                c->frame_aux_bytes = fb;
            }
            tgt_depth = c->frame_aux[0]; tgt_normal = c->frame_aux[1];
        }
    }
    if (c->cap_pairs == 0) {
        uint32_t init = n < (1u << 20) ? (1u << 20) : n;   // first guess; grows on demand
        s = ensure_pair_scratch(c, init);
        if (s != BGS_OK) return s;
    }
    const size_t frame_bytes = (size_t)W * H * format_bpp(out_format);
    void* target = c->frame;
    if (out_rgba && out_is_device_ptr) target = out_rgba;
    else {
        s = ensure_frame(c, frame_bytes);
        if (s != BGS_OK) return s;
        target = c->frame;
    }
    // async frames rendered into the library's own buffers alternate two device frames, so whatever consumes
    // frame k off the render stream (the D2H copy, the NCCL gather: both on the copy/comm stream) overlaps frame k+1
    const bool async_own = (st->flags & BGS_FLAG_ASYNC) && !(out_rgba && out_is_device_ptr);
    const bool async_host = async_own && out_rgba;
    // output mode of the blend kernels: format | mode << 8 (raster.cu)
    const bool blend_over = (st->flags & BGS_FLAG_BLEND_OVER_TARGET) != 0;
    const uint32_t raster_format = out_format | ((blend_over ? 2u : ((st->flags & BGS_FLAG_PREMULTIPLIED_OUT) ? 1u : 0u)) << 8);
    int fslot = 0;
    if (async_own) {
        if (blend_over) fslot = c->frame_toggle ^ 1;            // keep blending into the frame the previous call produced
        else { fslot = c->frame_toggle; c->frame_toggle ^= 1; }
        target = fslot ? c->frame_alt : c->frame;
    }

    // saturation-aware chunking: frames whose splats cover many tiles each (last frame: >= 32 pairs per visible splat
    // and >= 2^24 pairs: below that, one round is cheaper than the extra launches) run binning / tile sort /
    // blend in front-to-back rank rounds; the rounds after every tile has saturated emit nothing.
    // Quad-uv records only; BGS_FLAG_CHUNKS / _NO_CHUNKS force it.
    bool chunked = raster_mode == 0 && !want_aux && num_tiles <= CHUNK_MAX_TILES && !(st->flags & BGS_FLAG_NO_CHUNKS);
    if (chunked && !(st->flags & BGS_FLAG_CHUNKS))
        chunked = c->n_vis_hint > 0 && c->n_pairs_hint >= (c->last_chunks > 1 ? 3u << 22 : 1u << 24) &&
                  (uint64_t)c->n_pairs_hint >= (c->last_chunks > 1 ? 24ull : 32ull) * c->n_vis_hint;   // (hysteresis)
    const int rounds = chunked ? MAX_CHUNKS : 1;
    if (chunked && c->cap_state_tiles < num_tiles) {
        cudaFree(c->state); c->state = nullptr; c->cap_state_tiles = 0;
        CU(c, cudaMalloc(&c->state, (size_t)num_tiles * 256 * sizeof(float4)));
        c->cap_state_tiles = num_tiles;
    }

    for (int attempt = 0; attempt < 4; ++attempt) {
        s = ensure_arena(c, num_tiles);
        if (s != BGS_OK) return s;
        s = ensure_status(c, n, c->cap_pairs);
        if (s != BGS_OK) return s;
        cudaStream_t q = c->stream;
        uint32_t launches = 0;
        CU(c, cudaMemsetAsync(c->arena, 0, c->arena_bytes, q));   // counters, histograms, ranges: ~0.4 MB
        CU(c, cudaEventRecord(c->ev[0], q));
        // ---- stage 1: key-gen (+ stable compaction of the visible set)
        // compact mode: keys[0][slot], slot_ids[slot] = gaussian index, vals[0][slot] = slot (sort payload)
        // SORT_ALL    : keys[0][i], vals[0][i] = i (payload is the gaussian index itself)
        const bool by_slot = !sort_all;
        if (by_slot) {
            // the cooperative key-gen also produces the depth sort's digit histograms
            // (keys[1] = visibility-mask scratch until the sort's first pass overwrites it)
            CU(c, launch_keygen_coop(cloud->pos, n, fc, c->keys[1], c->keys[0], c->slot_ids, c->vals[0], c->kg_block_cnt,
                                     c->ctr, c->hist, depth_passes, (st->flags & BGS_FLAG_ASYNC) ? c->kg_grid_async : c->kg_grid, q));
        } else {
            launch_keygen_all(cloud->pos, n, fc, c->keys[0], c->vals[0], c->ctr, q);
        }
        ++launches;
        CU(c, cudaEventRecord(c->ev[1], q));
        // ---- stage 3 (compact mode): projection + colour in slot order on the second stream, concurrently
        //      with the depth sort (it only needs slot_ids); records land at recs[slot]
        const uint32_t n_hint = c->n_vis_hint ? c->n_vis_hint + c->n_vis_hint / 4 + 1024 : n;
        // Depth colouring needs sorted[1] / sorted[N-1]: the projection then waits for the sort
        const bool overlap = by_slot && st->rasterize_mode != BGS_RASTERIZE_DEPTH && !want_aux;
        if (overlap) CU(c, cudaEventRecord(c->ev_fork, q));
        // ---- stage 2: depth radix sort: all P = depth_bits / 8 digit places in ONE cooperative launch (enqueued before
        //      the projection so its one-CTA-per-SM grid becomes resident first; the projection fills the other half)
        CU(c, launch_radix_sort(c->keys[0], c->vals[0], c->keys[1], c->vals[1], &c->ctr->n_sort, n,
                                sort_all ? n : (c->n_vis_hint ? c->n_vis_hint : n), c->hist, sort_all ? 1 : 0, c->status_depth,
                                (size_t)radix_num_tiles(c->status_n) * 256, next_epoch(c), &c->ctr->barrier[1], depth_passes, 0,
                                nullptr, c->sm_count, c->rs_per_sm, q));
        ++launches;
        if (overlap) {
            CU(c, cudaStreamWaitEvent(c->stream2, c->ev_fork, 0));
            CU(c, cudaEventRecord(c->ev_p0, c->stream2));
            launch_project(cloud->f16, cloud->blocks, c->slot_ids, 1, c->ctr, fc, c->recs, raster_mode == 2 ? c->extra : nullptr,
                           n_hint < n ? n_hint : n, c->sm_count, c->cutoff_tab, nullptr, c->stream2);
            ++launches;
            CU(c, cudaEventRecord(c->ev_p1, c->stream2));
            CU(c, cudaEventRecord(c->ev_join, c->stream2));
        }
        const int cur = depth_passes & 1;
        c->depth_result = cur;
        CU(c, cudaEventRecord(c->ev[2], q));
        if (overlap) {
            CU(c, cudaStreamWaitEvent(q, c->ev_join, 0));
        } else {
            // ---- stage 3 after the sort: SORT_ALL (records by front-to-back rank) or Depth colouring (by slot)
            if (st->rasterize_mode == BGS_RASTERIZE_DEPTH || want_aux) {
                launch_depth_range(cloud->pos, n, c->vals[cur], by_slot ? c->slot_ids : nullptr, c->ctr, fc, q);
                ++launches;
            }
            CU(c, cudaEventRecord(c->ev_p0, q));
            launch_project(cloud->f16, cloud->blocks, by_slot ? c->slot_ids : c->vals[cur], by_slot ? 1 : 0, c->ctr, fc, c->recs,
                           raster_mode == 2 ? c->extra : nullptr, n_hint < n ? n_hint : n, c->sm_count, c->cutoff_tab,
                           want_aux ? c->aux : nullptr, q);
            ++launches;
            CU(c, cudaEventRecord(c->ev_p1, q));
        }
        CU(c, cudaEventRecord(c->ev[3], q));
        // ---- stage 4: tile binning -> stable tile-id sort -> ranges; stage 5: per-tile front-to-back blend.
        //      One round normally; `rounds` front-to-back rank rounds on chunked frames, each resuming the pixels'
        //      blend state, the last one writing the frame (identical pixels either way).
        // kernel variant picked from the previous frame's mean footprint (pairs per visible splat); results are identical
        const bool large_fp = c->n_vis_hint > 0 && (uint64_t)c->n_pairs_hint >= 8ull * c->n_vis_hint;
        int pcur = 0;
        for (int r = 0; r < rounds; ++r) {
            ChunkCounters* cc = &c->ctr->chunk[r];
            const uint32_t fa = rounds > 1 ? CHUNK_FRAC[r] : 0u, fb = rounds > 1 ? CHUNK_FRAC[r + 1] : 65536u;
            uint2* rng = c->ranges + (size_t)r * num_tiles;
            uint32_t* hist_r = c->hist + (size_t)(4 + 4 * r) * 256;
            // the depth sort's spare ping-pong buffers (N words each) hold the large-footprint queue
            CU(c, launch_bin_emit_coop(c->recs, by_slot ? c->vals[cur] : nullptr, c->ctr, cc, fa, fb, num_tiles,
                                       c->bin_block_cnt, tiles_x, c->cap_pairs, c->pkeys[0], c->pvals[0], c->keys[cur ^ 1],
                                       c->vals[cur ^ 1], c->cap_n, (st->flags & BGS_FLAG_ASYNC) ? c->bin_grid_async : c->bin_grid,
                                       c->d_sticky, q));
            ++launches;
            // stable tile-id sort of the pair list + per-tile ranges: histogram phase, both digit places and the range
            // build in ONE cooperative launch
            uint32_t p_hint = c->n_pairs_hint ? c->n_pairs_hint : c->cap_pairs;
            if (rounds > 1) p_hint = c->chunk_hint_valid ? c->chunk_pairs_hint[r] : c->cap_pairs;
            if (p_hint > c->cap_pairs) p_hint = c->cap_pairs;
            CU(c, launch_radix_sort(c->pkeys[0], c->pvals[0], c->pkeys[1], c->pvals[1], &cc->n_pairs, c->cap_pairs, p_hint, hist_r, 1,
                                    c->status_pairs, (size_t)radix_num_tiles(c->status_np) * 256, next_epoch(c), &cc->sort_barrier,
                                    tile_passes, 0, rng, c->sm_count, (st->flags & BGS_FLAG_ASYNC) ? SORT_CTAS_PER_SM_ASYNC : c->rs_per_sm, q));
            ++launches;
            pcur = tile_passes & 1;
            if (r + 1 == rounds) {
                // (chunked frames: the earlier rounds' blends are accounted to stage 4)
                CU(c, cudaEventRecord(c->ev[4], q));
                if (async_own && c->copy_pending[fslot]) CU(c, cudaStreamWaitEvent(q, c->ev_copied[fslot], 0));   // target free again
            }
            if (rounds == 1) {
                // the blend runs on the LOW-priority stream; the render stream resumes once it is done
                CU(c, cudaEventRecord(c->ev_front, q));
                CU(c, cudaStreamWaitEvent(c->stream_r, c->ev_front, 0));
                launch_raster(raster_mode, large_fp, c->recs, c->extra, c->pvals[pcur], rng, W, H, tiles_x, tiles_y, target, raster_format,
                              want_aux ? c->aux : nullptr, tgt_depth, tgt_normal, c->stream_r);
                CU(c, cudaEventRecord(c->ev_rdone, c->stream_r));
                CU(c, cudaStreamWaitEvent(q, c->ev_rdone, 0));
            } else
                launch_raster_round(c->recs, c->pvals[pcur], rng, W, H, tiles_x, tiles_y, target, raster_format, c->state,
                                    c->tile_done, &c->ctr->tiles_done, r == 0, r + 1 == rounds, q);
            ++launches;
        }
        c->pair_result = pcur;
        CU(c, cudaEventRecord(c->ev[5], q));
        CU(c, cudaEventRecord(c->ev_done, q));
        CU(c, cudaMemcpyAsync(c->h_ctr, c->ctr, sizeof(FrameCounters), cudaMemcpyDeviceToHost, q));
        CU(c, cudaMemcpyAsync(c->h_sticky, c->d_sticky, 4, cudaMemcpyDeviceToHost, q));
        if (async_own) CU(c, cudaEventRecord(c->ev_raster[fslot], q));
        if (async_host) {
            CU(c, cudaStreamWaitEvent(c->stream_copy, c->ev_raster[fslot], 0));
            CU(c, cudaMemcpyAsync(out_rgba, target, frame_bytes, cudaMemcpyDeviceToHost, c->stream_copy));
            CU(c, cudaEventRecord(c->ev_copied[fslot], c->stream_copy));
            c->copy_pending[fslot] = true;
        } else if (out_rgba && !out_is_device_ptr) {
            CU(c, cudaMemcpyAsync(out_rgba, target, frame_bytes, cudaMemcpyDeviceToHost, q));
            if (want_aux) {
                CU(c, cudaMemcpyAsync(out_depth, tgt_depth, frame_bytes, cudaMemcpyDeviceToHost, q));
                CU(c, cudaMemcpyAsync(out_normal, tgt_normal, frame_bytes, cudaMemcpyDeviceToHost, q));
            }
        }
        c->pend_cloud = cloud; c->pend_n = n; c->pend_fc = fc; c->pend_sort_all = sort_all; c->pend_by_slot = by_slot;
        c->pend_chunks = rounds;
        c->pend_tiles_x = tiles_x; c->pend_tiles_y = tiles_y; c->pend_W = W; c->pend_H = H; c->pend_target = target;
        if (st->flags & BGS_FLAG_ASYNC) {
            c->launches = launches;
            c->async_pending = true;
            c->have_frame = false;     // hooks need bgs_sync() first
            return BGS_OK;
        }
        CU(c, cudaStreamSynchronize(q));
        CU(c, cudaGetLastError());
        c->launches = launches;
        c->h_sticky[0] = 0;
        CU(c, cudaMemsetAsync(c->d_sticky, 0, 4, q));   // synchronous frames report their own overflow right here
        const bgs_status fs = finish_frame(c);
        if (fs == BGS_NOT_READY) continue;   // pair buffer grown: redo the frame
        return fs;
    }
    return fail(c, BGS_ENOMEM, "render: pair list kept overflowing");
}

bgs_status bgs_debug_sorted_entries(bgs_context* c, uint32_t* out) {
    if (!c || !out) return BGS_EINVAL;
    if (!c->have_frame || !c->last_cloud) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    CU(c, cudaSetDevice(c->device));
    const uint32_t n = c->last_cloud->n, n_vis = c->stats.n_visible;
    const uint32_t n_sorted = c->last_sort_all ? n : n_vis;
    std::vector<uint32_t> k(n_sorted), v(n_sorted);
    CU(c, cudaMemcpy(k.data(), c->keys[c->depth_result], (size_t)n_sorted * 4, cudaMemcpyDeviceToHost));
    CU(c, cudaMemcpy(v.data(), c->vals[c->depth_result], (size_t)n_sorted * 4, cudaMemcpyDeviceToHost));
    if (c->last_by_slot) {   // the sort's payload is the compact slot: map it to the gaussian index
        std::vector<uint32_t> ids(n_sorted);
        CU(c, cudaMemcpy(ids.data(), c->slot_ids, (size_t)n_sorted * 4, cudaMemcpyDeviceToHost));
        for (uint32_t i = 0; i < n_sorted; ++i) v[i] = ids[v[i]];
    }
    for (uint32_t i = 0; i < n_sorted; ++i) { out[2 * i] = k[i]; out[2 * i + 1] = v[i]; }
    if (!c->last_sort_all) {
        // culled tail: key = all-ones >> shift, indices ascending (what a stable sort leaves there)
        uint32_t* flags = nullptr;
        CU(c, cudaMalloc(&flags, (size_t)n * 4));
        launch_culled_flags(c->last_cloud->pos, n, c->last_fc, flags, c->stream);
        std::vector<uint32_t> f(n);
        cudaError_t e = cudaMemcpyAsync(f.data(), flags, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        cudaFree(flags);
        if (e != cudaSuccess) return fail(c, BGS_ECUDA, "debug_sorted_entries: %s", cudaGetErrorString(e));
        const uint32_t culled_key = 0xFFFFFFFFu >> c->last_fc.key_shift;
        uint32_t at = n_vis;
        for (uint32_t i = 0; i < n; ++i)
            if (f[i]) {
                if (at >= n) return fail(c, BGS_ECUDA, "debug_sorted_entries: visible/culled counts disagree");
                out[2 * at] = culled_key; out[2 * at + 1] = i; ++at;
            }
        if (at != n) return fail(c, BGS_ECUDA, "debug_sorted_entries: visible/culled counts disagree");
    }
    return BGS_OK;
}

bgs_status bgs_debug_tile_ranges(bgs_context* c, uint32_t* start_end) {
    if (!c || !start_end) return BGS_EINVAL;
    if (!c->have_frame) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    if (c->last_chunks > 1) return fail(c, BGS_NOT_READY, "the last frame was binned in %d rounds: set BGS_FLAG_NO_CHUNKS for the tile hooks", c->last_chunks);
    CU(c, cudaSetDevice(c->device));
    const size_t tiles = (size_t)c->stats.tiles_x * c->stats.tiles_y;
    CU(c, cudaMemcpy(start_end, c->ranges, tiles * 8, cudaMemcpyDeviceToHost));
    // device form: (~start, end), (0, 0) for an empty tile (the sort's last pass builds them with atomicMax)
    for (size_t t = 0; t < tiles; ++t) {
        if (start_end[2 * t + 1] == 0u) start_end[2 * t] = 0u;
        else start_end[2 * t] = ~start_end[2 * t];
    }
    return BGS_OK;
}

bgs_status bgs_debug_tile_entries(bgs_context* c, uint32_t* ranks, uint64_t capacity) {
    if (!c || !ranks) return BGS_EINVAL;
    if (!c->have_frame) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    if (c->last_chunks > 1) return fail(c, BGS_NOT_READY, "the last frame was binned in %d rounds: set BGS_FLAG_NO_CHUNKS for the tile hooks", c->last_chunks);
    CU(c, cudaSetDevice(c->device));
    const uint64_t cnt = c->stats.n_pairs < capacity ? c->stats.n_pairs : capacity;
    CU(c, cudaMemcpy(ranks, c->pvals[c->pair_result], (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    if (c->last_by_slot) {   // pair payload = record index = compact slot: convert to front-to-back rank
        const uint32_t n_vis = c->stats.n_visible;
        std::vector<uint32_t> perm(n_vis), inv(n_vis);
        CU(c, cudaMemcpy(perm.data(), c->vals[c->depth_result], (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
        for (uint32_t r = 0; r < n_vis; ++r) inv[perm[n_vis - 1 - r]] = r;
        for (uint64_t i = 0; i < cnt; ++i) ranks[i] = ranks[i] < n_vis ? inv[ranks[i]] : 0xFFFFFFFFu;
    }
    return BGS_OK;
}

bgs_status bgs_debug_projected(bgs_context* c, float* records, uint32_t* rank_to_index) {
    if (!c) return BGS_EINVAL;
    if (!c->have_frame) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    CU(c, cudaSetDevice(c->device));
    const uint32_t n_vis = c->stats.n_visible;
    std::vector<uint32_t> v(n_vis), ids;
    CU(c, cudaMemcpy(v.data(), c->vals[c->depth_result], (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
    if (c->last_by_slot) {
        ids.resize(n_vis);
        CU(c, cudaMemcpy(ids.data(), c->slot_ids, (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
    }
    if (records) {
        std::vector<SplatRec> tmp(n_vis);
        CU(c, cudaMemcpy(tmp.data(), c->recs, (size_t)n_vis * sizeof(SplatRec), cudaMemcpyDeviceToHost));
        for (uint32_t r = 0; r < n_vis; ++r) {
            const uint32_t ri = c->last_by_slot ? v[n_vis - 1 - r] : r;   // rank -> record index
            memcpy(records + (size_t)r * 12, &tmp[ri], sizeof(SplatRec));
        }
    }
    if (rank_to_index)
        for (uint32_t r = 0; r < n_vis; ++r) rank_to_index[r] = c->last_by_slot ? ids[v[n_vis - 1 - r]] : v[n_vis - 1 - r];
    return BGS_OK;
}

bgs_status bgs_frame_stats_get(bgs_context* c, bgs_frame_stats* out) {
    if (!c || !out) return BGS_EINVAL;
    if (!c->have_frame) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    *out = c->stats;
    return BGS_OK;
}

bgs_status bgs_stage_times_us(bgs_context* c, float out[6]) {
    if (!c || !out) return BGS_EINVAL;
    if (!c->have_frame) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    if (!c->stage_valid) {
        for (int i = 0; i < 5; ++i) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, c->ev[i], c->ev[i + 1]);
            c->stage_us[i] = ms * 1000.f;
        }
        {   // the projection may overlap the sort (second stream): report its own duration
            float pms = 0.f;
            cudaEventElapsedTime(&pms, c->ev_p0, c->ev_p1);
            c->stage_us[2] = pms * 1000.f;
        }
        float ms = 0.f;
        cudaEventElapsedTime(&ms, c->ev[0], c->ev[5]);
        c->stage_us[5] = ms * 1000.f;
        c->stage_valid = true;
    }
    for (int i = 0; i < 6; ++i) out[i] = c->stage_us[i];
    return BGS_OK;
}

// gather.cc: where to run the gather of `local_frame`.  A library-owned frame of an async render is consumed on the
// copy/comm stream (after its raster), so the next frame on the render stream overlaps the transfer; anything else
// runs on the render stream.  `*slot` >= 0 -> call bgs_internal_gather_end_ afterwards.
cudaStream_t bgs_internal_gather_begin_(bgs_context* c, const void* local_frame, int* slot) {
    *slot = -1;
    if (!c) return nullptr;
    for (int k = 0; k < 2; ++k) {
        const void* f = k ? c->frame_alt : c->frame;
        if (f && f == local_frame && c->async_pending) {
            if (cudaStreamWaitEvent(c->stream_copy, c->ev_raster[k], 0) != cudaSuccess) return c->stream;
            *slot = k;
            return c->stream_copy;
        }
    }
    return c->stream;
}
void bgs_internal_gather_end_(bgs_context* c, int slot) {
    if (!c || slot < 0) return;
    if (cudaEventRecord(c->ev_copied[slot], c->stream_copy) == cudaSuccess) c->copy_pending[slot] = true;
}

const char* bgs_last_error(const bgs_context* c) { return c ? c->err : "null context"; }
void* bgs_context_stream(bgs_context* c) { return c ? (void*)c->stream : nullptr; }
void* bgs_context_copy_stream(bgs_context* c) { return c ? (void*)c->stream_copy : nullptr; }
const void* bgs_frame_device_ptr(bgs_context* c) {
    if (!c) return nullptr;
    return c->have_frame ? c->last_frame : (c->async_pending ? c->pend_target : nullptr);
}
uint32_t bgs_last_launch_count(const bgs_context* c) { return c ? c->launches : 0; }

}  // extern "C"
