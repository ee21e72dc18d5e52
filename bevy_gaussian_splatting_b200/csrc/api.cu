// api.cu -- the extern "C" boundary of libbgs (include/bgs.h): contexts, clouds, the per-view
// frame (stage orchestration on one CUDA stream), parity/debug hooks, stage timing.
//
// No PyTorch, no wgpu, no CPU fallback: every stage is a hand-written sm_90a kernel.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <atomic>
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
// select.cu
uint32_t select_num_buckets(uint32_t n);
int select_sort_passes(uint32_t n_buckets);
void launch_select_keys(const float4* pos, uint32_t n, float radius, uint32_t n_buckets, uint32_t* keys, uint32_t* vals,
                        uint32_t* n_sort, cudaStream_t stream);
void launch_select_count(const float4* pos, const uint32_t* ids, const uint2* ranges, uint32_t n, float radius, uint32_t n_buckets,
                         float r2, uint32_t threshold, float4* spos, float* pos_w, float* block_w, uint32_t block_stride,
                         uint32_t* selected, cudaStream_t stream);
void launch_select_fill(uint32_t n, float v, float* pos_w, float* block_w, uint32_t block_stride, cudaStream_t stream);
// mesh_select.cu
size_t mesh_words_bytes();
size_t mesh_rec_bytes();
void launch_mesh_setup(const float* verts, const uint32_t* idx, uint32_t nt, void* bin_rec, void* bin_box, void* glob_rec, void* words,
                       cudaStream_t stream);
void launch_mesh_levels(const void* bin_box, const void* words_host, void* words, cudaStream_t stream);
void mesh_pick_level(const void* words_host, int* level, uint64_t* pairs, uint32_t* cells);
void launch_mesh_emit(const void* bin_box, const void* words_host, int level, uint32_t* keys, uint32_t* vals, void* words,
                      cudaStream_t stream);
uint32_t* mesh_words_pairs(void* words);
uint32_t* mesh_words_barrier(void* words);
uint32_t* mesh_words_inside(void* words);
uint32_t mesh_words_n_bin(const void* words_host);
void launch_mesh_count(const float4* pos, uint32_t n, const float* mesh_from_cloud, const void* bin_rec, const void* glob_rec,
                       const uint32_t* cell_tri, const uint2* ranges, const void* words_host, int level, uint32_t mode, float* pos_w,
                       float* block_w, uint32_t block_stride, void* words, cudaStream_t stream);
// particles.cu
void launch_particle_step(void* behaviors, uint32_t count, float dt, float4* pos, void* blocks, uint32_t block_stride,
                          cudaStream_t stream);
// subset.cu
uint32_t subset_num_ctas(uint32_t n);
void launch_subset_count(const float4* pos, uint32_t n, uint32_t* mask, uint32_t* cta_cnt, uint32_t* total, cudaStream_t stream);
void launch_subset_scatter(bool f16, const void* pos, const void* blocks, uint32_t n, const uint32_t* mask, const uint32_t* cta_off,
                           void* out_pos, void* out_blocks, cudaStream_t stream);
void launch_subset_gather(bool f16, const void* pos, const void* blocks, const uint32_t* idx, uint32_t k, void* out_pos,
                          void* out_blocks, cudaStream_t stream);
void launch_unpack(bool f16, const void* blocks, uint32_t lo, uint32_t m, void* sh, void* rot, void* so, cudaStream_t stream);
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
    // enqueued writes (particle steps): ev_write marks the last one, on whichever context's stream it was queued; every
    // later reader or writer waits for it on the device.  Created by the first step; `stepped` is set once it exists,
    // so a cloud that is never stepped costs its frames nothing
    cudaEvent_t ev_write = nullptr;
    std::atomic<bool> stepped{false};
};

// A ParticleBehaviors asset resident on one GPU: count 64 B records (bgs_particle_behavior), read and written by the step
struct bgs_particles {
    int device;
    uint32_t count;
    int64_t max_index;            // largest active gaussian index (-1: none is active)
    void* d = nullptr;            // count * 64 B
    cudaEvent_t ev_write = nullptr;   // the last step of these behaviours (recorded on the stepping context's stream)
};

// A grow-only device buffer.  grow() replaces a buffer smaller than `want` bytes by one of exactly `want` bytes, zeroed
// on the render stream when asked; a failed grow leaves it empty.  Its owner (the context) releases it on destruction.
namespace {
template <class T>
struct DevBuf {
    T* p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    bgs_status grow(bgs_context* c, size_t want, bool zero);
    void release() { cudaFree(p); p = nullptr; bytes = 0; }
};
}  // namespace

// What the host knows of a frame it has enqueued: the context keeps the last one enqueued (`pend`) and, once its
// counters are back, the last one completed (`last`, what the debug hooks read).
struct FrameFacts {
    const bgs_cloud* cloud = nullptr;   // (nulled if the cloud is destroyed meanwhile)
    uint32_t n = 0;                     // gaussians in the cloud (a snapshot: the cloud may be gone by the time it is read)
    FrameConsts fc = {};
    bool sort_all = false;
    bool by_slot = false;               // records indexed by compact slot (else by front-to-back rank)
    int rounds = 1;                     // binning rounds
    int tiles_x = 0, tiles_y = 0, W = 0, H = 0;
    const void* target = nullptr;       // the device frame the blend wrote
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
    cudaStream_t stream_copy = nullptr;   // copy/comm stream: D2H copies and gathers of queued frames (default priority)
    cudaEvent_t ev[6] = {};               // stage boundaries (timed)
    cudaEvent_t ev_p0 = nullptr, ev_p1 = nullptr;   // the projection's own start / end (timed)
    cudaEvent_t ev_front = nullptr, ev_rdone = nullptr, ev_fork = nullptr, ev_join = nullptr, ev_done = nullptr;
    cudaEvent_t ev_raster[2] = {nullptr, nullptr}, ev_copied[2] = {nullptr, nullptr};
    uint32_t n_vis_hint = 0;          // last frame's visible count (sizes the projection grid)
    uint32_t n_pairs_hint = 0;        // last frame's pair count (picks the pair sort's tile size); on chunked
                                      // frames an ESTIMATE of what one round would have emitted
    uint32_t chunk_pairs_hint[MAX_CHUNKS] = {};   // last chunked frame's pairs per round (pair sort tile size)
    bool chunk_hint_valid = false;
    char err[512] = {0};

    // scratch sized by the cloud (grow-only; cap_n gaussians)
    uint32_t cap_n = 0;
    DevBuf<uint32_t> keys[2], vals[2];
    DevBuf<uint32_t> slot_ids;        // compact slot -> gaussian index (key-gen output, index order)
    DevBuf<SplatRec> recs;
    DevBuf<float4> extra;             // 4 x float4 per record: 2DGS + USE_AABB only (allocated on first use)
    DevBuf<float4> aux;               // 2 x float4 per record: depth / normal colour sources (bgs_render_aux only)
    DevBuf<void> frame_aux[2];        // depth / normal frames when bgs_render_aux delivers to host memory
    // scratch sized by the pair capacity (grow-only; cap_pairs pairs)
    uint32_t cap_pairs = 0;
    DevBuf<uint32_t> pkeys[2], pvals[2];
    DevBuf<float4> state;             // per-pixel blend state between rounds (tile-major), tiles * 256 * 16 B
    // zeroed-per-frame arena: counters | hist | keygen CTA counts | bin CTA counts | ranges | done bytes
    DevBuf<uint8_t> arena;
    uint32_t arena_tiles = 0;
    // look-back status rows of the two sorts (64-bit epoch-tagged words, cleared once at allocation)
    DevBuf<void> status_depth;        // [4][tiles(status_n)][256]
    DevBuf<void> status_pairs;        // [4][tiles(status_np)][256]
    uint32_t status_n = 0, status_np = 0;
    // bgs_cloud_select_sparse's own words, zeroed per call: sort count | sort barrier | selected | digit histograms |
    // per-bucket ranges (the sort and the record buffer are the frame's, see bgs_cloud_select_sparse)
    DevBuf<uint8_t> select_scratch;
    // bgs_cloud_select_in_mesh's own scratch (never the frame's): words | vertices | indices | binned records | binned
    // boxes | global records, and the pair side: digit histograms | per-cell ranges | pair keys / values x 2
    DevBuf<uint8_t> mesh_tri, mesh_pairs;
    bool async_pending = false;        // a BGS_FLAG_ASYNC frame has been enqueued and not yet completed
    bool step_pending = false;         // a particle step has been enqueued since the last bgs_sync
    FrameCounters* ctr = nullptr;
    uint32_t* hist = nullptr;          // [8 + 4 * MAX_CHUNKS][256]: depth passes 0..3, pair passes 4..7 (round 0), 8 + 4r.. (round r)
    uint32_t* kg_block_cnt = nullptr;  // [kg_grid]: keygen_coop's per-CTA visible counts
    uint32_t* bin_block_cnt = nullptr; // [bin_grid][3]: bin_emit_coop's per-CTA pair / medium / large counts
    uint2* ranges = nullptr;           // per tile (~start, end) into the sorted pair list (0, 0 = empty)
    unsigned char* tile_done = nullptr;   // per tile: saturated (chunked frames)
    // async frames delivered to host memory alternate the two frames so frame k's D2H copy (copy stream) overlaps
    // frame k+1's kernels
    DevBuf<void> frames[2];
    int frame_toggle = 0;
    bool copy_pending[2] = {false, false};
    FrameCounters* h_ctr = nullptr;    // pinned
    float* cutoff_tab = nullptr;       // adaptive cutoff of every f16 opacity value (project.cu)
    // largest n_pairs_needed of ANY frame since the last bgs_sync / synchronous render (device word outside the
    // per-frame arena + its pinned copy): a queued async frame that overflowed the pair buffer is never missed
    uint32_t* d_sticky = nullptr;
    uint32_t* h_sticky = nullptr;      // [0] the copy of *d_sticky, [1] a selection's selected / inside count
    // bgs_cloud_download_*'s two pinned bounce buffers (2 x 30 MB, allocated by the first download, kept until the
    // context goes): one chunk's planes each, so the host's copy of one chunk overlaps the device-to-host copy of the next
    uint8_t* h_bounce = nullptr;
    std::vector<bgs_cloud*> clouds;    // clouds uploaded through this context (their ctx is nulled on destroy)

    FrameFacts pend, last;
    bool have_frame = false;           // `last` is valid (for the debug hooks)
    int depth_result = 0, pair_result = 0;   // which ping-pong buffer holds the sorted result
    bgs_frame_stats stats = {};
    float stage_us[6] = {0, 0, 0, 0, 0, 0};
    bool stage_valid = false;
    uint32_t launches = 0;

    // every stream with its priority (0 = highest, 1, 2 = lowest, -1 = the default) and every event with whether it is
    // timed: bgs_context_create creates them, bgs_context_destroy destroys them
    template <class F> void each_stream(F f) { f(stream, 0); f(stream2, 1); f(stream_r, 2); f(stream_copy, -1); }
    template <class F> void each_event(F f) {
        for (cudaEvent_t& e : ev) f(e, true);
        f(ev_p0, true); f(ev_p1, true);
        for (cudaEvent_t* e : {&ev_front, &ev_rdone, &ev_fork, &ev_join, &ev_done, &ev_raster[0], &ev_raster[1],
                               &ev_copied[0], &ev_copied[1]})
            f(*e, false);
    }
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

#define TRY(call)                     \
    do {                              \
        const bgs_status s_ = (call); \
        if (s_ != BGS_OK) return s_;  \
    } while (0)

template <class T>
bgs_status DevBuf<T>::grow(bgs_context* c, size_t want, bool zero) {
    if (want <= bytes) return BGS_OK;
    release();
    void* np = nullptr;
    cudaError_t e = cudaMalloc(&np, want);
    if (e == cudaSuccess && zero) e = cudaMemsetAsync(np, 0, want, c->stream);
    if (e != cudaSuccess) {
        cudaFree(np);
        return fail(c, e == cudaErrorMemoryAllocation ? BGS_ENOMEM : BGS_ECUDA, "allocating %zu bytes of device scratch: %s",
                    want, cudaGetErrorString(e));
    }
    p = static_cast<T*>(np);
    bytes = want;
    return BGS_OK;
}

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
    c->cap_n = 0;
    for (int i = 0; i < 2; ++i) {
        // (>= 1024 words: keys[1] doubles as key-gen's visibility-mask scratch, one word per 32 gaussians rounded up to a tile)
        TRY(c->keys[i].grow(c, (size_t)std::max(n, 1024u) * 4, false));
        TRY(c->vals[i].grow(c, (size_t)std::max(n, 1024u) * 4, false));
    }
    TRY(c->slot_ids.grow(c, (size_t)n * 4, false));
    TRY(c->recs.grow(c, (size_t)n * sizeof(SplatRec), false));
    c->cap_n = n;
    return BGS_OK;
}

bgs_status ensure_pair_scratch(bgs_context* c, uint32_t pairs) {
    if (pairs <= c->cap_pairs) return BGS_OK;
    c->cap_pairs = 0;
    for (int i = 0; i < 2; ++i) {
        // +64 words: the raster's 16 B-granular bulk copies may read a few entries past the last pair
        TRY(c->pkeys[i].grow(c, ((size_t)pairs + 64) * 4, false));
        TRY(c->pvals[i].grow(c, ((size_t)pairs + 64) * 4, false));
    }
    c->cap_pairs = pairs;
    return BGS_OK;
}

// A frame (one round) needed `needed` pairs: BGS_OK if they fit, else the pair buffer grows (x1.25 head-room) and the
// frame must be rendered again (BGS_NOT_READY), or BGS_ENOMEM at the 2^30 limit.
bgs_status grow_pairs(bgs_context* c, uint32_t needed) {
    if (needed <= c->cap_pairs) return BGS_OK;
    uint64_t want = (uint64_t)needed + needed / 4 + 1024;
    if (want >= (1ull << 30)) want = (1ull << 30) - 1;
    if (needed >= LB_VMASK || want <= c->cap_pairs) return fail(c, BGS_ENOMEM, "render: frame needs >= 2^30 (splat, tile) pairs");
    TRY(ensure_pair_scratch(c, (uint32_t)want));
    return BGS_NOT_READY;
}

bgs_status ensure_arena(bgs_context* c, uint32_t tiles) {
    if (c->arena.p && tiles <= c->arena_tiles) return BGS_OK;
    tiles = std::max(tiles, c->arena_tiles);
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
    TRY(c->arena.grow(c, off, false));
    c->ctr = reinterpret_cast<FrameCounters*>(c->arena.p + o_ctr);
    c->hist = reinterpret_cast<uint32_t*>(c->arena.p + o_hist);
    c->kg_block_cnt = reinterpret_cast<uint32_t*>(c->arena.p + o_kgc);
    c->bin_block_cnt = reinterpret_cast<uint32_t*>(c->arena.p + o_binc);
    c->ranges = reinterpret_cast<uint2*>(c->arena.p + o_rng);
    c->tile_done = c->arena.p + o_done;
    c->arena_tiles = tiles;
    return BGS_OK;
}

// look-back status rows of a sort of up to `capacity` entries: 4 passes x tiles x 256 digits x 8 B, epoch-tagged
// (radix.cu), so they are cleared exactly once -- when allocated -- and never again
bgs_status ensure_status(bgs_context* c, DevBuf<void>& rows, uint32_t& rows_capacity, uint32_t capacity) {
    if (capacity <= rows_capacity) return BGS_OK;
    rows_capacity = 0;
    TRY(rows.grow(c, (size_t)4 * radix_num_tiles(capacity) * 256 * 8, true));
    rows_capacity = capacity;
    return BGS_OK;
}

uint32_t next_epoch(bgs_context* c) {
    if (++c->sort_epoch >= (1u << 30)) {     // (2^30 sorts later) start over from clean rows
        for (DevBuf<void>* s : {&c->status_depth, &c->status_pairs})
            if (s->p) cudaMemsetAsync(s->p, 0, s->bytes, c->stream);
        c->sort_epoch = 1;
    }
    return c->sort_epoch;
}

size_t format_bpp(uint32_t f) { return f == BGS_FORMAT_RGBA32F ? 16 : (f == BGS_FORMAT_RGBA16F ? 8 : 4); }

// Every choice a frame's launches depend on beyond the frame itself: made from the settings, the previous frame's
// counts (the hints) and the context's grids and capacities.  plan_frame makes no CUDA call and changes nothing.
struct FramePlan {
    int raster_mode;        // 0 = quad-uv falloff (USE_OBB, 3DGS and 2DGS), 1 = 3DGS conic (USE_AABB), 2 = 2DGS ray-splat (USE_AABB)
    int rounds;             // binning rounds: 1, or MAX_CHUNKS on a chunked frame
    bool large_fp;          // blend variant for large footprints (results are identical)
    bool by_slot;           // compact mode: records at recs[slot] (else SORT_ALL: by front-to-back rank)
    bool depth_range;       // Depth colouring / aux frames: the projection needs sorted[1] / sorted[N-1]
    bool overlap;           // the projection runs on the second stream beside the depth sort
    int depth_passes, tile_passes;   // digit places of the depth sort and of the tile-id sort
    uint32_t kg_grid, bin_grid;      // cooperative key-gen / binning CTAs
    int pair_sort_per_sm;            // radix-sort CTAs per SM of the tile-id sort
    uint32_t depth_hint;             // entries the depth sort plans for
    uint32_t n_hint;                 // records the projection grid plans for
    uint32_t pair_hint[MAX_CHUNKS];  // pairs each round's tile-id sort plans for
};

FramePlan plan_frame(const bgs_context* c, const bgs_settings* st, bool want_aux, uint32_t num_tiles, uint32_t n) {
    FramePlan p;
    const bool queued = (st->flags & BGS_FLAG_ASYNC) != 0;
    p.raster_mode = !st->aabb ? 0 : (st->gaussian_mode == BGS_GAUSSIAN_3D ? 1 : 2);
    // saturation-aware chunking: frames whose splats cover many tiles each (last frame: >= 32 pairs per visible splat
    // and >= 2^24 pairs: below that, one round is cheaper than the extra launches) run binning / tile sort /
    // blend in front-to-back rank rounds; the rounds after every tile has saturated emit nothing.
    // Quad-uv records only; BGS_FLAG_CHUNKS / _NO_CHUNKS force it.
    bool chunked = p.raster_mode == 0 && !want_aux && num_tiles <= CHUNK_MAX_TILES && !(st->flags & BGS_FLAG_NO_CHUNKS);
    if (chunked && !(st->flags & BGS_FLAG_CHUNKS))
        chunked = c->n_vis_hint > 0 && c->n_pairs_hint >= (c->last.rounds > 1 ? 3u << 22 : 1u << 24) &&
                  (uint64_t)c->n_pairs_hint >= (c->last.rounds > 1 ? 24ull : 32ull) * c->n_vis_hint;   // (hysteresis)
    p.rounds = chunked ? MAX_CHUNKS : 1;
    // kernel variant picked from the previous frame's mean footprint (pairs per visible splat)
    p.large_fp = c->n_vis_hint > 0 && (uint64_t)c->n_pairs_hint >= 8ull * c->n_vis_hint;
    p.by_slot = !(st->flags & BGS_FLAG_SORT_ALL);
    p.depth_range = st->rasterize_mode == BGS_RASTERIZE_DEPTH || want_aux;
    p.overlap = p.by_slot && !p.depth_range;
    p.depth_passes = (int)st->radix_sort_depth_bits / 8;
    p.tile_passes = pair_passes(num_tiles);
    p.kg_grid = queued ? c->kg_grid_async : c->kg_grid;
    p.bin_grid = queued ? c->bin_grid_async : c->bin_grid;
    p.pair_sort_per_sm = queued ? SORT_CTAS_PER_SM_ASYNC : c->rs_per_sm;
    p.depth_hint = !p.by_slot ? n : (c->n_vis_hint ? c->n_vis_hint : n);
    p.n_hint = std::min(c->n_vis_hint ? c->n_vis_hint + c->n_vis_hint / 4 + 1024 : n, n);
    for (int r = 0; r < p.rounds; ++r) {
        uint32_t h = c->n_pairs_hint ? c->n_pairs_hint : c->cap_pairs;
        if (p.rounds > 1) h = c->chunk_hint_valid ? c->chunk_pairs_hint[r] : c->cap_pairs;
        p.pair_hint[r] = std::min(h, c->cap_pairs);
    }
    return p;
}

// Where a frame's pixels go.
struct FrameOut {
    void* rgba = nullptr;               // the blend's target (device): the caller's frame or one of the library's
    void* depth = nullptr;              // bgs_render_aux's depth / normal targets (device)
    void* normal = nullptr;
    uint32_t raster_format = 0;         // output mode of the blend kernels: format | mode << 8 (raster.cu)
    size_t bytes = 0;                   // of one frame
    int slot = -1;                      // a queued frame in the library's own frames: which of the two (else -1)
    void* host_rgba = nullptr;          // host frames the result is copied to
    void* host_depth = nullptr;
    void* host_normal = nullptr;
};

// the caller's device frames, or the library's own (grown on demand)
bgs_status frame_out(bgs_context* c, const bgs_settings* st, uint32_t format, size_t bytes, void* out_rgba,
                     int out_is_device_ptr, bool want_aux, void* out_depth, void* out_normal, FrameOut* o) {
    const bool blend_over = (st->flags & BGS_FLAG_BLEND_OVER_TARGET) != 0;
    o->raster_format = format | ((blend_over ? 2u : ((st->flags & BGS_FLAG_PREMULTIPLIED_OUT) ? 1u : 0u)) << 8);
    o->bytes = bytes;
    if (out_rgba && out_is_device_ptr) {
        o->rgba = out_rgba;
    } else {
        for (int k = 0; k < 2; ++k) {
            if (bytes <= c->frames[k].bytes) continue;
            TRY(c->frames[k].grow(c, bytes, true));      // (BGS_FLAG_BLEND_OVER_TARGET reads the target)
            c->copy_pending[k] = false;
        }
        // async frames rendered into the library's own buffers alternate two device frames, so whatever consumes
        // frame k off the render stream (the D2H copy, the NCCL gather: both on the copy/comm stream) overlaps frame k+1
        if (st->flags & BGS_FLAG_ASYNC) {
            if (blend_over) o->slot = c->frame_toggle ^ 1;            // keep blending into the frame the previous call produced
            else { o->slot = c->frame_toggle; c->frame_toggle ^= 1; }
        }
        o->rgba = c->frames[std::max(o->slot, 0)].p;
        o->host_rgba = out_rgba;
    }
    if (!want_aux) return BGS_OK;
    if (out_is_device_ptr) { o->depth = out_depth; o->normal = out_normal; return BGS_OK; }
    for (int k = 0; k < 2; ++k) TRY(c->frame_aux[k].grow(c, bytes, true));
    o->depth = c->frame_aux[0].p; o->normal = c->frame_aux[1].p;
    o->host_depth = out_depth; o->host_normal = out_normal;
    return BGS_OK;
}

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
    const int prio[3] = {prio_hi, (prio_lo + prio_hi) / 2, prio_lo};
    c->each_stream([&](cudaStream_t& s, int rank) {
        if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, rank < 0 ? 0 : prio[rank]);
    });
    c->each_event([&](cudaEvent_t& ev, bool timed) {
        if (e == cudaSuccess) e = timed ? cudaEventCreate(&ev) : cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    });
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
    c->each_stream([](cudaStream_t& s, int) { if (s) cudaStreamSynchronize(s); });
    c->each_event([](cudaEvent_t& ev, bool) { if (ev) cudaEventDestroy(ev); });
    c->each_stream([](cudaStream_t& s, int) { if (s) cudaStreamDestroy(s); });
    if (c->h_ctr) cudaFreeHost(c->h_ctr);
    if (c->h_sticky) cudaFreeHost(c->h_sticky);
    if (c->h_bounce) cudaFreeHost(c->h_bounce);
    cudaFree(c->d_sticky);
    cudaFree(c->cutoff_tab);
    delete c;   // (releases every DevBuf)
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
            if (c->pend.cloud == cl || c->last.cloud == cl) {
                if (c->async_pending || c->pend.cloud == cl) c->each_stream([](cudaStream_t& s, int) { cudaStreamSynchronize(s); });
                if (c->pend.cloud == cl) { c->pend.cloud = nullptr; c->pend.n = 0; }
                if (c->last.cloud == cl) { c->last.cloud = nullptr; c->have_frame = false; }
            }
            c->clouds.erase(std::remove(c->clouds.begin(), c->clouds.end(), cl), c->clouds.end());
        }
    }
    if (cl->ev_write) {   // particle steps still queued on any context write the planes
        cudaEventSynchronize(cl->ev_write);
        cudaEventDestroy(cl->ev_write);
    }
    cudaFree(cl->pos); cudaFree(cl->blocks);
    delete cl;
}

// Bookkeeping once a frame's counters are back on the host (sync render, or bgs_sync after async ones).
static bgs_status finish_frame(bgs_context* c) {
    const int chunks = c->pend.rounds;
    uint32_t needed = 0;
    uint64_t emitted = 0;
    for (int r = 0; r < chunks; ++r) {
        const ChunkCounters& cc = c->h_ctr->chunk[r];
        needed = cc.n_pairs_needed > needed ? cc.n_pairs_needed : needed;
        emitted += cc.n_pairs;
    }
    TRY(grow_pairs(c, needed));   // (the pair list of one round did not fit: the caller redoes the frame)
    c->last = c->pend;
    c->have_frame = true;
    c->stage_valid = false;
    c->stats.n = c->last.n; c->stats.n_visible = c->h_ctr->n_vis; c->stats.n_pairs = emitted;
    c->stats.rounds = (uint32_t)chunks; c->stats.tiles_saturated = c->h_ctr->tiles_done;
    c->stats.tiles_x = (uint32_t)c->last.tiles_x; c->stats.tiles_y = (uint32_t)c->last.tiles_y;
    c->stats.width = (uint32_t)c->last.W; c->stats.height = (uint32_t)c->last.H;
    c->n_vis_hint = c->h_ctr->n_vis;
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
    c->err[0] = 0;
    return BGS_OK;
}

bgs_status bgs_sync(bgs_context* c) {
    if (!c) return BGS_EINVAL;
    if (!c->async_pending && !c->step_pending) return BGS_OK;
    CU(c, cudaSetDevice(c->device));
    c->step_pending = false;
    if (!c->async_pending) {   // only particle steps were queued: no frame to account for
        CU(c, cudaStreamSynchronize(c->stream));
        CU(c, cudaGetLastError());
        return BGS_OK;
    }
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaStreamSynchronize(c->stream_copy));
    c->copy_pending[0] = c->copy_pending[1] = false;
    CU(c, cudaGetLastError());
    c->async_pending = false;
    // the sticky maximum covers EVERY frame queued since the last sync, not just the last one (whose counters are
    // in h_ctr): any of them that needed more pairs than the buffer holds was blended from a truncated list
    const uint32_t worst = c->h_sticky[0];
    c->h_sticky[0] = 0;
    CU(c, cudaMemsetAsync(c->d_sticky, 0, 4, c->stream));
    const bgs_status s = finish_frame(c);
    if (s == BGS_NOT_READY) return fail(c, BGS_NOT_READY, "an async frame outgrew the pair buffer (now grown): render the frames queued since the last bgs_sync again");
    if (s != BGS_OK) return s;
    const bgs_status gs = grow_pairs(c, worst);
    if (gs == BGS_NOT_READY) {
        c->have_frame = false;
        return fail(c, BGS_NOT_READY, "an earlier async frame (not the last one) outgrew the pair buffer (now grown): every frame queued since the last bgs_sync may be truncated, render them again");
    }
    return gs;
}

static bgs_status check_render(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                               const bgs_settings* st, uint32_t out_format, bool want_aux) {
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
    return BGS_OK;
}

static FrameConsts frame_consts(const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                                const bgs_settings* st, bool want_aux) {
    const int W = (int)view->viewport[2], H = (int)view->viewport[3];
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
    fc.Wi = W; fc.Hi = H; fc.tiles_x = (W + TILE_PX - 1) / TILE_PX; fc.tiles_y = (H + TILE_PX - 1) / TILE_PX;
    fc.n_cloud = cloud->n;
    fc.aux = want_aux ? 1u : 0u;
    fc.cov_pre = cloud->cov ? 1u : 0u;
    memcpy(fc.aabb_min, uni->aabb_min, 12); memcpy(fc.aabb_max, uni->aabb_max, 12);
    static const float kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    fc.model_identity = memcmp(uni->transform, kIdentity, 64) == 0 ? 1u : 0u;   // (-0.0 entries take the general path)
    return fc;
}

// Enqueues one attempt at a frame: every launch of the plan, the counters' read-back and the copy-out.
static bgs_status enqueue_frame(bgs_context* c, const bgs_cloud* cloud, const FrameConsts& fc, const FramePlan& p,
                                const FrameOut& o) {
    const uint32_t n = cloud->n;
    const uint32_t num_tiles = (uint32_t)fc.tiles_x * (uint32_t)fc.tiles_y;
    cudaStream_t q = c->stream;
    uint32_t launches = 0;
    // a stepped cloud: the frame reads the positions of every step enqueued before it, on any context
    if (cloud->stepped.load(std::memory_order_acquire)) CU(c, cudaStreamWaitEvent(q, cloud->ev_write, 0));
    CU(c, cudaMemsetAsync(c->arena.p, 0, c->arena.bytes, q));   // counters, histograms, ranges: ~0.4 MB
    CU(c, cudaEventRecord(c->ev[0], q));
    // ---- stage 1: key-gen (+ stable compaction of the visible set)
    // compact mode: keys[0][slot], slot_ids[slot] = gaussian index, vals[0][slot] = slot (sort payload)
    // SORT_ALL    : keys[0][i], vals[0][i] = i (payload is the gaussian index itself)
    if (p.by_slot) {
        // the cooperative key-gen also produces the depth sort's digit histograms
        // (keys[1] = visibility-mask scratch until the sort's first pass overwrites it)
        CU(c, launch_keygen_coop(cloud->pos, n, fc, c->keys[1].p, c->keys[0].p, c->slot_ids.p, c->vals[0].p, c->kg_block_cnt,
                                 c->ctr, c->hist, p.depth_passes, p.kg_grid, q));
    } else {
        launch_keygen_all(cloud->pos, n, fc, c->keys[0].p, c->vals[0].p, c->ctr, q);
    }
    ++launches;
    CU(c, cudaEventRecord(c->ev[1], q));
    if (p.overlap) CU(c, cudaEventRecord(c->ev_fork, q));
    // ---- stage 2: depth radix sort: all P = depth_bits / 8 digit places in ONE cooperative launch (enqueued before
    //      the projection so its one-CTA-per-SM grid becomes resident first; the projection fills the other half)
    CU(c, launch_radix_sort(c->keys[0].p, c->vals[0].p, c->keys[1].p, c->vals[1].p, &c->ctr->n_sort, n, p.depth_hint,
                            c->hist, p.by_slot ? 0 : 1, c->status_depth.p, (size_t)radix_num_tiles(c->status_n) * 256,
                            next_epoch(c), &c->ctr->barrier[1], p.depth_passes, 0, nullptr, c->sm_count, c->rs_per_sm, q));
    ++launches;
    const int cur = p.depth_passes & 1;
    c->depth_result = cur;
    CU(c, cudaEventRecord(c->ev[2], q));
    // ---- stage 3: projection + colour.  Compact mode: in slot order on the second stream, concurrently with the depth
    //      sort (it only needs slot_ids); records land at recs[slot].  After the sort: SORT_ALL (records by front-to-back
    //      rank), or Depth colouring / aux frames (by slot), which need the depth range of the sorted set first
    const cudaStream_t ps = p.overlap ? c->stream2 : q;
    if (p.overlap) CU(c, cudaStreamWaitEvent(c->stream2, c->ev_fork, 0));
    if (p.depth_range) {
        launch_depth_range(cloud->pos, n, c->vals[cur].p, p.by_slot ? c->slot_ids.p : nullptr, c->ctr, fc, q);
        ++launches;
    }
    CU(c, cudaEventRecord(c->ev_p0, ps));
    launch_project(cloud->f16, cloud->blocks, p.by_slot ? c->slot_ids.p : c->vals[cur].p, p.by_slot ? 1 : 0, c->ctr, fc,
                   c->recs.p, p.raster_mode == 2 ? c->extra.p : nullptr, p.n_hint, c->sm_count, c->cutoff_tab,
                   fc.aux ? c->aux.p : nullptr, ps);
    ++launches;
    CU(c, cudaEventRecord(c->ev_p1, ps));
    if (p.overlap) {
        CU(c, cudaEventRecord(c->ev_join, c->stream2));
        CU(c, cudaStreamWaitEvent(q, c->ev_join, 0));
    }
    CU(c, cudaEventRecord(c->ev[3], q));
    // ---- stage 4: tile binning -> stable tile-id sort -> ranges; stage 5: per-tile front-to-back blend.
    //      One round normally; `rounds` front-to-back rank rounds on chunked frames, each resuming the pixels'
    //      blend state, the last one writing the frame (identical pixels either way).
    int pcur = 0;
    for (int r = 0; r < p.rounds; ++r) {
        ChunkCounters* cc = &c->ctr->chunk[r];
        const uint32_t fa = p.rounds > 1 ? CHUNK_FRAC[r] : 0u, fb = p.rounds > 1 ? CHUNK_FRAC[r + 1] : 65536u;
        uint2* rng = c->ranges + (size_t)r * num_tiles;
        uint32_t* hist_r = c->hist + (size_t)(4 + 4 * r) * 256;
        // the depth sort's spare ping-pong buffers (N words each) hold the large-footprint queue
        CU(c, launch_bin_emit_coop(c->recs.p, p.by_slot ? c->vals[cur].p : nullptr, c->ctr, cc, fa, fb, num_tiles,
                                   c->bin_block_cnt, fc.tiles_x, c->cap_pairs, c->pkeys[0].p, c->pvals[0].p,
                                   c->keys[cur ^ 1].p, c->vals[cur ^ 1].p, c->cap_n, p.bin_grid, c->d_sticky, q));
        ++launches;
        // stable tile-id sort of the pair list + per-tile ranges: histogram phase, both digit places and the range
        // build in ONE cooperative launch
        CU(c, launch_radix_sort(c->pkeys[0].p, c->pvals[0].p, c->pkeys[1].p, c->pvals[1].p, &cc->n_pairs, c->cap_pairs,
                                p.pair_hint[r], hist_r, 1, c->status_pairs.p, (size_t)radix_num_tiles(c->status_np) * 256,
                                next_epoch(c), &cc->sort_barrier, p.tile_passes, 0, rng, c->sm_count, p.pair_sort_per_sm, q));
        ++launches;
        pcur = p.tile_passes & 1;
        if (r + 1 == p.rounds) {
            // (chunked frames: the earlier rounds' blends are accounted to stage 4)
            CU(c, cudaEventRecord(c->ev[4], q));
            if (o.slot >= 0 && c->copy_pending[o.slot]) CU(c, cudaStreamWaitEvent(q, c->ev_copied[o.slot], 0));   // target free again
        }
        if (p.rounds == 1) {
            // the blend runs on the LOW-priority stream; the render stream resumes once it is done
            CU(c, cudaEventRecord(c->ev_front, q));
            CU(c, cudaStreamWaitEvent(c->stream_r, c->ev_front, 0));
            launch_raster(p.raster_mode, p.large_fp, c->recs.p, c->extra.p, c->pvals[pcur].p, rng, fc.Wi, fc.Hi, fc.tiles_x,
                          fc.tiles_y, o.rgba, o.raster_format, fc.aux ? c->aux.p : nullptr, o.depth, o.normal, c->stream_r);
            CU(c, cudaEventRecord(c->ev_rdone, c->stream_r));
            CU(c, cudaStreamWaitEvent(q, c->ev_rdone, 0));
        } else
            launch_raster_round(c->recs.p, c->pvals[pcur].p, rng, fc.Wi, fc.Hi, fc.tiles_x, fc.tiles_y, o.rgba, o.raster_format,
                                c->state.p, c->tile_done, &c->ctr->tiles_done, r == 0, r + 1 == p.rounds, q);
        ++launches;
    }
    c->pair_result = pcur;
    CU(c, cudaEventRecord(c->ev[5], q));
    CU(c, cudaEventRecord(c->ev_done, q));
    CU(c, cudaMemcpyAsync(c->h_ctr, c->ctr, sizeof(FrameCounters), cudaMemcpyDeviceToHost, q));
    CU(c, cudaMemcpyAsync(c->h_sticky, c->d_sticky, 4, cudaMemcpyDeviceToHost, q));
    if (o.slot >= 0) CU(c, cudaEventRecord(c->ev_raster[o.slot], q));
    if (o.slot >= 0 && o.host_rgba) {
        CU(c, cudaStreamWaitEvent(c->stream_copy, c->ev_raster[o.slot], 0));
        CU(c, cudaMemcpyAsync(o.host_rgba, o.rgba, o.bytes, cudaMemcpyDeviceToHost, c->stream_copy));
        CU(c, cudaEventRecord(c->ev_copied[o.slot], c->stream_copy));
        c->copy_pending[o.slot] = true;
    } else if (o.host_rgba) {
        CU(c, cudaMemcpyAsync(o.host_rgba, o.rgba, o.bytes, cudaMemcpyDeviceToHost, q));
        if (o.host_depth) {
            CU(c, cudaMemcpyAsync(o.host_depth, o.depth, o.bytes, cudaMemcpyDeviceToHost, q));
            CU(c, cudaMemcpyAsync(o.host_normal, o.normal, o.bytes, cudaMemcpyDeviceToHost, q));
        }
    }
    c->pend = {cloud, n, fc, !p.by_slot, p.by_slot, p.rounds, fc.tiles_x, fc.tiles_y, fc.Wi, fc.Hi, o.rgba};
    c->launches = launches;
    return BGS_OK;
}

static bgs_status render_impl(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                              const bgs_settings* st, void* out_rgba, uint32_t out_format, int out_is_device_ptr,
                              bool want_aux, void* out_depth, void* out_normal) {
    if (!c) return BGS_EINVAL;
    TRY(check_render(c, cloud, view, uni, st, out_format, want_aux));
    CU(c, cudaSetDevice(c->device));
    if (c->async_pending && !(st->flags & BGS_FLAG_ASYNC)) {
        // a synchronous render after queued frames completes them first; their failure (including an overflowed
        // pair list = BGS_NOT_READY) is the caller's to see, so this frame is not rendered on top of it
        TRY(bgs_sync(c));
    }
    const FrameConsts fc = frame_consts(cloud, view, uni, st, want_aux);
    const uint32_t n = cloud->n, num_tiles = (uint32_t)fc.tiles_x * (uint32_t)fc.tiles_y;
    TRY(ensure_cloud_scratch(c, n));
    if (c->cap_pairs == 0) TRY(ensure_pair_scratch(c, std::max(n, 1u << 20)));   // first guess; grows on demand
    FrameOut o;
    TRY(frame_out(c, st, out_format, (size_t)fc.Wi * fc.Hi * format_bpp(out_format), out_rgba, out_is_device_ptr, want_aux,
                  out_depth, out_normal, &o));
    for (int attempt = 0; attempt < 4; ++attempt) {
        const FramePlan p = plan_frame(c, st, want_aux, num_tiles, n);   // (each attempt: the pair hints read cap_pairs)
        if (p.raster_mode == 2) TRY(c->extra.grow(c, (size_t)c->cap_n * 64, false));
        if (want_aux) TRY(c->aux.grow(c, (size_t)c->cap_n * 32, false));
        if (p.rounds > 1) TRY(c->state.grow(c, (size_t)num_tiles * 256 * sizeof(float4), false));
        TRY(ensure_arena(c, num_tiles));
        TRY(ensure_status(c, c->status_depth, c->status_n, n));
        TRY(ensure_status(c, c->status_pairs, c->status_np, c->cap_pairs));
        TRY(enqueue_frame(c, cloud, fc, p, o));
        if (st->flags & BGS_FLAG_ASYNC) {
            c->async_pending = true;
            c->have_frame = false;     // hooks need bgs_sync() first
            return BGS_OK;
        }
        CU(c, cudaStreamSynchronize(c->stream));
        CU(c, cudaGetLastError());
        c->h_sticky[0] = 0;
        CU(c, cudaMemsetAsync(c->d_sticky, 0, 4, c->stream));   // synchronous frames report their own overflow right here
        const bgs_status fs = finish_frame(c);
        if (fs != BGS_NOT_READY) return fs;   // (BGS_NOT_READY: pair buffer grown, redo the frame)
    }
    return fail(c, BGS_ENOMEM, "render: pair list kept overflowing");
}

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

// ---- selection edits of a resident cloud (select.cu).  The visibility lane lives twice on the device: the position
// plane's .w (what key-gen streams) and the first 16 B of each gaussian-major block (what the projection reads): every
// write updates both.

// The particle steps enqueued on any context before a call that reads or writes the cloud on this context's stream.
static bgs_status wait_cloud_steps(bgs_context* c, const bgs_cloud* cl) {
    if (cl->stepped.load(std::memory_order_acquire)) CU(c, cudaStreamWaitEvent(c->stream, cl->ev_write, 0));
    return BGS_OK;
}

// Before a selection writes a cloud: this context's queued frames are completed (their failure is returned, as a
// synchronous render does), and so are the queued frames of every other context on the cloud's GPU, which may read it.
// Particle steps queued on any context come first on the device (the writer runs on this context's stream).
static bgs_status quiesce_for_write(bgs_context* c, const bgs_cloud* cl) {
    if (c->async_pending) TRY(bgs_sync(c));
    TRY(wait_cloud_steps(c, cl));
    std::lock_guard<std::mutex> lk(g_registry_mu);
    for (bgs_context* o : g_contexts)
        if (o != c && o->device == cl->device && o->async_pending)
            o->each_stream([](cudaStream_t& s, int) { cudaStreamSynchronize(s); });
    return BGS_OK;
}

static size_t block_bytes(const bgs_cloud* cl) { return cl->f16 ? 128 : 256; }

bgs_status bgs_cloud_select_sparse(bgs_context* c, bgs_cloud* cl, float radius, uint32_t threshold, uint32_t* out_selected) {
    if (!c) return BGS_EINVAL;
    if (!cl) return fail(c, BGS_EINVAL, "select_sparse: null cloud");
    if (!(radius >= 0.0f) || std::isinf(radius)) return fail(c, BGS_EINVAL, "select_sparse: radius must be finite and >= 0");
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "select_sparse: cloud lives on another device");
    CU(c, cudaSetDevice(c->device));
    TRY(quiesce_for_write(c, cl));
    const uint32_t n = cl->n;
    const float r2 = radius * radius;
    float* pos_w = reinterpret_cast<float*>(cl->pos) + 3;
    float* block_w = reinterpret_cast<float*>(cl->blocks) + 3;
    const uint32_t stride = (uint32_t)(block_bytes(cl) / 4);
    cudaStream_t q = c->stream;
    uint32_t selected = 0;
    if (threshold == 0u || r2 == 0.0f) {
        // no count can reach a threshold of 0; no distance is below a radius whose square is 0 (every count is 0)
        selected = threshold == 0u ? 0u : n;
        launch_select_fill(n, threshold == 0u ? 0.0f : 1.0f, pos_w, block_w, stride, q);
        CU(c, cudaGetLastError());
        CU(c, cudaStreamSynchronize(q));
    } else {
        // the frame's scratch: key / value ping-pong buffers and depth-sort status rows (the sort), the record buffer
        // (positions in bucket order).  The debug hooks lose the last frame; the hints the next frame plans from stay.
        TRY(ensure_cloud_scratch(c, n));
        TRY(ensure_status(c, c->status_depth, c->status_n, n));
        const uint32_t nb = select_num_buckets(n);
        const int passes = select_sort_passes(nb);
        const size_t o_hist = 256, o_rng = o_hist + 4 * 256 * 4;
        TRY(c->select_scratch.grow(c, o_rng + ((size_t)nb + 1) * sizeof(uint2), false));
        c->have_frame = false;
        uint32_t* words = reinterpret_cast<uint32_t*>(c->select_scratch.p);   // [0] sort count, [1] barrier, [2] selected
        uint32_t* hist = reinterpret_cast<uint32_t*>(c->select_scratch.p + o_hist);
        uint2* ranges = reinterpret_cast<uint2*>(c->select_scratch.p + o_rng);   // nb + 1: the sentinel key's too
        CU(c, cudaMemsetAsync(c->select_scratch.p, 0, o_rng + ((size_t)nb + 1) * sizeof(uint2), q));
        launch_select_keys(cl->pos, n, radius, nb, c->keys[0].p, c->vals[0].p, &words[0], q);
        CU(c, cudaGetLastError());
        CU(c, launch_radix_sort(c->keys[0].p, c->vals[0].p, c->keys[1].p, c->vals[1].p, &words[0], n, n, hist, 1,
                                c->status_depth.p, (size_t)radix_num_tiles(c->status_n) * 256, next_epoch(c), &words[1], passes,
                                0, ranges, c->sm_count, c->rs_per_sm, q));
        launch_select_count(cl->pos, c->vals[passes & 1].p, ranges, n, radius, nb, r2, threshold,
                            reinterpret_cast<float4*>(c->recs.p), pos_w, block_w, stride, &words[2], q);
        CU(c, cudaGetLastError());
        CU(c, cudaMemcpyAsync(c->h_sticky + 1, &words[2], 4, cudaMemcpyDeviceToHost, q));
        CU(c, cudaStreamSynchronize(q));
        selected = c->h_sticky[1];
    }
    if (out_selected) *out_selected = selected;
    return BGS_OK;
}

bgs_status bgs_cloud_visibility_get(bgs_context* c, const bgs_cloud* cl, float* out_vis) {
    if (!c) return BGS_EINVAL;
    if (!cl || !out_vis) return fail(c, BGS_EINVAL, "visibility_get: null cloud or array");
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "visibility_get: cloud lives on another device");
    CU(c, cudaSetDevice(c->device));
    TRY(wait_cloud_steps(c, cl));
    CU(c, cudaMemcpy2DAsync(out_vis, 4, reinterpret_cast<const char*>(cl->pos) + 12, 16, 4, cl->n, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

bgs_status bgs_cloud_visibility_set(bgs_context* c, bgs_cloud* cl, const float* vis) {
    if (!c) return BGS_EINVAL;
    if (!cl || !vis) return fail(c, BGS_EINVAL, "visibility_set: null cloud or array");
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "visibility_set: cloud lives on another device");
    CU(c, cudaSetDevice(c->device));
    TRY(quiesce_for_write(c, cl));
    CU(c, cudaMemcpy2DAsync(reinterpret_cast<char*>(cl->pos) + 12, 16, vis, 4, 4, cl->n, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpy2DAsync(reinterpret_cast<char*>(cl->blocks) + 12, block_bytes(cl), vis, 4, 4, cl->n, cudaMemcpyHostToDevice,
                            c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

bgs_status bgs_cloud_select_in_mesh(bgs_context* c, bgs_cloud* cl, const float* vertices, uint32_t nv, const uint32_t* indices,
                                    uint32_t nt, const float* mesh_from_cloud, uint32_t mode, uint32_t* out_inside) {
    if (!c) return BGS_EINVAL;
    if (!cl) return fail(c, BGS_EINVAL, "select_in_mesh: null cloud");
    if (nt > 0 && (!vertices || !indices)) return fail(c, BGS_EINVAL, "select_in_mesh: null vertices or indices");
    if (mode != BGS_SELECT_REPLACE && mode != BGS_SELECT_ADD) return fail(c, BGS_EINVAL, "select_in_mesh: unknown mode %u", mode);
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "select_in_mesh: cloud lives on another device");
    for (size_t k = 0; k < (size_t)nt * 3; ++k)
        if (indices[k] >= nv) return fail(c, BGS_EINVAL, "select_in_mesh: index %u of triangle %zu is >= %u vertices", indices[k], k / 3, nv);
    if (nt >= (1u << 26)) return fail(c, BGS_ENOMEM, "select_in_mesh: more than 2^26 triangles");
    static const float identity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const float* M = mesh_from_cloud ? mesh_from_cloud : identity;
    CU(c, cudaSetDevice(c->device));
    TRY(quiesce_for_write(c, cl));
    const uint32_t n = cl->n;
    float* pos_w = reinterpret_cast<float*>(cl->pos) + 3;
    float* block_w = reinterpret_cast<float*>(cl->blocks) + 3;
    const uint32_t stride = (uint32_t)(block_bytes(cl) / 4);
    cudaStream_t q = c->stream;

    // triangle side: setup (records, classes, grid bounds)
    const size_t o_v = 256, o_i = align_up(o_v + (size_t)nv * 12, 256), o_br = align_up(o_i + (size_t)nt * 12, 256);
    const size_t o_bb = o_br + (size_t)nt * mesh_rec_bytes(), o_gr = o_bb + (size_t)nt * 32, tri_bytes = o_gr + (size_t)nt * mesh_rec_bytes();
    TRY(c->mesh_tri.grow(c, tri_bytes, false));
    uint8_t* tb = c->mesh_tri.p;
    void* words = tb;
    std::vector<unsigned long long> wh_buf((mesh_words_bytes() + 7) / 8);
    void* wh = wh_buf.data();
    CU(c, cudaMemsetAsync(words, 0, 256, q));
    if (nt > 0) {
        CU(c, cudaMemcpyAsync(tb + o_v, vertices, (size_t)nv * 12, cudaMemcpyHostToDevice, q));
        CU(c, cudaMemcpyAsync(tb + o_i, indices, (size_t)nt * 12, cudaMemcpyHostToDevice, q));
        launch_mesh_setup(reinterpret_cast<const float*>(tb + o_v), reinterpret_cast<const uint32_t*>(tb + o_i), nt, tb + o_br,
                          tb + o_bb, tb + o_gr, words, q);
        CU(c, cudaGetLastError());
    }
    CU(c, cudaMemcpyAsync(wh, words, mesh_words_bytes(), cudaMemcpyDeviceToHost, q));
    CU(c, cudaStreamSynchronize(q));

    // grid side: the level, the pairs, their sort by cell
    int level = -1;
    const uint32_t* cell_tri = nullptr;
    const uint2* ranges = nullptr;
    if (mesh_words_n_bin(wh) > 0) {
        launch_mesh_levels(tb + o_bb, wh, words, q);
        CU(c, cudaGetLastError());
        CU(c, cudaMemcpyAsync(wh, words, mesh_words_bytes(), cudaMemcpyDeviceToHost, q));
        CU(c, cudaStreamSynchronize(q));
        uint64_t pairs64 = 0;
        uint32_t cells = 0;
        mesh_pick_level(wh, &level, &pairs64, &cells);
        const uint32_t pairs = (uint32_t)pairs64;
        const size_t o_rng = 4 * 256 * 4, o_k0 = align_up(o_rng + (size_t)cells * 8, 256), pw = align_up((size_t)pairs * 4, 256);
        TRY(c->mesh_pairs.grow(c, o_k0 + 4 * pw, false));
        TRY(ensure_status(c, c->status_pairs, c->status_np, pairs));
        uint8_t* pb = c->mesh_pairs.p;
        uint32_t* k0 = reinterpret_cast<uint32_t*>(pb + o_k0);
        uint32_t* v0 = reinterpret_cast<uint32_t*>(pb + o_k0 + pw);
        uint32_t* k1 = reinterpret_cast<uint32_t*>(pb + o_k0 + 2 * pw);
        uint32_t* v1 = reinterpret_cast<uint32_t*>(pb + o_k0 + 3 * pw);
        uint2* rng = reinterpret_cast<uint2*>(pb + o_rng);
        CU(c, cudaMemsetAsync(pb, 0, o_k0, q));
        launch_mesh_emit(tb + o_bb, wh, level, k0, v0, words, q);
        CU(c, cudaGetLastError());
        const int passes = pair_passes(cells);
        CU(c, launch_radix_sort(k0, v0, k1, v1, mesh_words_pairs(words), pairs, pairs, reinterpret_cast<uint32_t*>(pb), 1,
                                c->status_pairs.p, (size_t)radix_num_tiles(c->status_np) * 256, next_epoch(c),
                                mesh_words_barrier(words), passes, 0, rng, c->sm_count, c->rs_per_sm, q));
        cell_tri = (passes & 1) ? v1 : v0;
        ranges = rng;
    }

    // point side: the count and the lane
    launch_mesh_count(cl->pos, n, M, tb + o_br, tb + o_gr, cell_tri, ranges, wh, level, mode, pos_w, block_w, stride, words, q);
    CU(c, cudaGetLastError());
    CU(c, cudaMemcpyAsync(c->h_sticky + 1, mesh_words_inside(words), 4, cudaMemcpyDeviceToHost, q));
    CU(c, cudaStreamSynchronize(q));
    if (out_inside) *out_inside = c->h_sticky[1];
    return BGS_OK;
}

// ---- particle behaviours (particles.cu).  The step is enqueued, never drained: it waits on the device for whatever
// may still read the positions (the queued frames of every context on the GPU: each context's ev_done marks its last
// frame; earlier steps of the cloud and of the behaviours), and marks itself on the cloud and the behaviours for
// whatever comes after.

bgs_status bgs_particles_create(bgs_context* c, const bgs_particle_behavior* behaviors, uint32_t count, bgs_particles** out) {
    if (!c || !out) return BGS_EINVAL;
    *out = nullptr;
    if (!behaviors) return fail(c, BGS_EINVAL, "particles_create: null behaviours");
    if (count == 0 || count >= (1u << 30)) return fail(c, BGS_EINVAL, "particles_create: count must be in [1, 2^30)");
    static_assert(sizeof(bgs_particle_behavior) == 64, "ParticleBehavior is 64 B");
    std::vector<uint32_t> active;
    active.reserve(count);
    for (uint32_t i = 0; i < count; ++i)
        if (behaviors[i].indices[0] < 0x80000000u) active.push_back(behaviors[i].indices[0]);
    std::sort(active.begin(), active.end());
    const auto dup = std::adjacent_find(active.begin(), active.end());
    if (dup != active.end()) return fail(c, BGS_EINVAL, "particles_create: two active behaviours name gaussian %u", *dup);
    CU(c, cudaSetDevice(c->device));
    bgs_particles* p = new (std::nothrow) bgs_particles();
    if (!p) return BGS_ENOMEM;
    p->device = c->device;
    p->count = count;
    p->max_index = active.empty() ? -1 : (int64_t)active.back();
    cudaError_t e = cudaMalloc(&p->d, (size_t)count * 64);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_write, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMemcpyAsync(p->d, behaviors, (size_t)count * 64, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        bgs_particles_destroy(p);
        return fail(c, e == cudaErrorMemoryAllocation ? BGS_ENOMEM : BGS_ECUDA, "particles_create: %s", cudaGetErrorString(e));
    }
    *out = p;
    return BGS_OK;
}

bgs_status bgs_particles_get(bgs_context* c, const bgs_particles* p, bgs_particle_behavior* out) {
    if (!c) return BGS_EINVAL;
    if (!p || !out) return fail(c, BGS_EINVAL, "particles_get: null behaviours or array");
    if (p->device != c->device) return fail(c, BGS_EINVAL, "particles_get: behaviours live on another device");
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamWaitEvent(c->stream, p->ev_write, 0));   // every step of these behaviours, on any context
    CU(c, cudaMemcpyAsync(out, p->d, (size_t)p->count * 64, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

void bgs_particles_destroy(bgs_particles* p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->ev_write) {   // steps still queued on any context read and write the records
        cudaEventSynchronize(p->ev_write);
        cudaEventDestroy(p->ev_write);
    }
    cudaFree(p->d);
    delete p;
}

bgs_status bgs_cloud_particles_step(bgs_context* c, bgs_cloud* cl, bgs_particles* p, float delta_time) {
    if (!c) return BGS_EINVAL;
    if (!cl || !p) return fail(c, BGS_EINVAL, "particles_step: null cloud or behaviours");
    if (!std::isfinite(delta_time)) return fail(c, BGS_EINVAL, "particles_step: delta_time must be finite");
    if (cl->device != c->device || p->device != c->device)
        return fail(c, BGS_EINVAL, "particles_step: cloud or behaviours live on another device");
    if (p->max_index >= (int64_t)cl->n)
        return fail(c, BGS_EINVAL, "particles_step: behaviour names gaussian %lld of a cloud of %u", (long long)p->max_index, cl->n);
    CU(c, cudaSetDevice(c->device));
    cudaStream_t q = c->stream;
    {
        // (under the registry lock: another context's step of the same cloud or behaviours waits and records in turn)
        std::lock_guard<std::mutex> lk(g_registry_mu);
        if (!cl->ev_write) CU(c, cudaEventCreateWithFlags(&cl->ev_write, cudaEventDisableTiming));
        for (bgs_context* o : g_contexts)
            if (o != c && o->device == c->device) CU(c, cudaStreamWaitEvent(q, o->ev_done, 0));
        if (cl->stepped.load(std::memory_order_relaxed)) CU(c, cudaStreamWaitEvent(q, cl->ev_write, 0));
        CU(c, cudaStreamWaitEvent(q, p->ev_write, 0));
        launch_particle_step(p->d, p->count, delta_time, cl->pos, cl->blocks, (uint32_t)(block_bytes(cl) / 16), q);
        CU(c, cudaGetLastError());
        CU(c, cudaEventRecord(cl->ev_write, q));
        CU(c, cudaEventRecord(p->ev_write, q));
        cl->stepped.store(true, std::memory_order_release);
    }
    c->step_pending = true;
    return BGS_OK;
}

bgs_status bgs_cloud_positions_get(bgs_context* c, const bgs_cloud* cl, float* out_pos_vis) {
    if (!c) return BGS_EINVAL;
    if (!cl || !out_pos_vis) return fail(c, BGS_EINVAL, "positions_get: null cloud or array");
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "positions_get: cloud lives on another device");
    CU(c, cudaSetDevice(c->device));
    TRY(wait_cloud_steps(c, cl));
    CU(c, cudaMemcpyAsync(out_pos_vis, cl->pos, (size_t)cl->n * 16, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

// ---- subset and download (subset.cu).  Both only read the source cloud, after every particle step queued on it (on
// the device, like visibility_get); neither drains another context's frames.  Their scratch is their own, allocated and
// released on the render stream within the call (stream-ordered: no device-wide synchronisation), so the frame's
// buffers, the debug hooks and the next frame's plan are untouched.

// Device scratch of one call, released on the stream when it goes out of scope.
namespace {
struct StreamScratch {
    void* p = nullptr;
    cudaStream_t q;
    explicit StreamScratch(cudaStream_t s) : q(s) {}
    StreamScratch(const StreamScratch&) = delete;
    StreamScratch& operator=(const StreamScratch&) = delete;
    ~StreamScratch() { if (p) cudaFreeAsync(p, q); }
    cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, q); }
};
}  // namespace

bgs_status bgs_cloud_subset(bgs_context* c, const bgs_cloud* cl, const uint32_t* indices, uint32_t k, bgs_cloud** out,
                            uint32_t* out_n) {
    if (!c) return BGS_EINVAL;
    if (out) *out = nullptr;
    if (!cl || !out) return fail(c, BGS_EINVAL, "subset: null cloud or out");
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "subset: cloud lives on another device");
    if (!indices && k != 0) return fail(c, BGS_EINVAL, "subset: selection mode (indices == NULL) takes k == 0");
    if (indices && (k == 0 || k >= (1u << 30))) return fail(c, BGS_EINVAL, "subset: k must be in [1, 2^30)");
    for (uint32_t j = 0; indices && j < k; ++j)
        if (indices[j] >= cl->n) return fail(c, BGS_EINVAL, "subset: index %u at %u is >= the cloud's %u gaussians", indices[j], j, cl->n);
    CU(c, cudaSetDevice(c->device));
    TRY(wait_cloud_steps(c, cl));
    cudaStream_t q = c->stream;
    const uint32_t n = cl->n;
    StreamScratch scratch(q);
    // selection mode: mask words | CTA counts (-> offsets) | the total
    const size_t o_cnt = align_up((size_t)(n + 31) / 32 * 4, 256), o_tot = align_up(o_cnt + (size_t)subset_num_ctas(n) * 4, 256);
    uint32_t kept = k;
    if (!indices) {
        CU(c, scratch.alloc(o_tot + 4));
        uint8_t* s = static_cast<uint8_t*>(scratch.p);
        launch_subset_count(cl->pos, n, reinterpret_cast<uint32_t*>(s), reinterpret_cast<uint32_t*>(s + o_cnt),
                            reinterpret_cast<uint32_t*>(s + o_tot), q);
        CU(c, cudaGetLastError());
        CU(c, cudaMemcpyAsync(c->h_sticky + 1, s + o_tot, 4, cudaMemcpyDeviceToHost, q));
        CU(c, cudaStreamSynchronize(q));
        kept = c->h_sticky[1];
        if (kept == 0) {
            if (out_n) *out_n = 0;
            return BGS_OK;
        }
    } else {
        CU(c, scratch.alloc((size_t)k * 4));
        CU(c, cudaMemcpyAsync(scratch.p, indices, (size_t)k * 4, cudaMemcpyHostToDevice, q));
    }
    bgs_cloud* nc = new (std::nothrow) bgs_cloud();
    if (!nc) return fail(c, BGS_ENOMEM, "subset: out of host memory");
    nc->ctx = c; nc->device = c->device; nc->n = kept; nc->f16 = cl->f16; nc->cov = cl->cov;
    nc->pos = nullptr; nc->blocks = nullptr;
    cudaError_t e = cudaMalloc(&nc->pos, (size_t)kept * 16);
    if (e == cudaSuccess) e = cudaMalloc(&nc->blocks, (size_t)kept * block_bytes(cl));
    if (e == cudaSuccess) {
        if (!indices) {
            const uint8_t* s = static_cast<const uint8_t*>(scratch.p);
            launch_subset_scatter(cl->f16, cl->pos, cl->blocks, n, reinterpret_cast<const uint32_t*>(s),
                                  reinterpret_cast<const uint32_t*>(s + o_cnt), nc->pos, nc->blocks, q);
        } else {
            launch_subset_gather(cl->f16, cl->pos, cl->blocks, static_cast<const uint32_t*>(scratch.p), k, nc->pos, nc->blocks, q);
        }
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(q);
    if (e != cudaSuccess) {
        cudaFree(nc->pos); cudaFree(nc->blocks);
        delete nc;
        return fail(c, e == cudaErrorMemoryAllocation ? BGS_ENOMEM : BGS_ECUDA, "subset: %s", cudaGetErrorString(e));
    }
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);
        c->clouds.push_back(nc);
    }
    *out = nc;
    if (out_n) *out_n = kept;
    return BGS_OK;
}

// gaussians per chunk of a download: the device staging arrays hold one chunk (f32: 28 MB), each of the context's two
// pinned bounce buffers one chunk's four planes (f32: 30 MB)
constexpr uint32_t DOWNLOAD_CHUNK = 1u << 17;
constexpr size_t DOWNLOAD_BOUNCE_BYTES = (size_t)DOWNLOAD_CHUNK * (16 + 192 + 16 + 16);

// Per chunk: unpack into device staging, copy the chunk's position plane and the staged planes to a pinned bounce
// buffer, and -- while the next chunk goes the same way into the other bounce buffer -- copy it into the caller's arrays.
static bgs_status download_common(bgs_context* c, const bgs_cloud* cl, bool f16, float* pos_vis, void* sh, void* rot, void* so) {
    if (!c) return BGS_EINVAL;
    if (!cl || !pos_vis || !sh || !rot || (!f16 && !so)) return fail(c, BGS_EINVAL, "download: null cloud or plane pointer");
    if (cl->device != c->device) return fail(c, BGS_EINVAL, "download: cloud lives on another device");
    if (cl->f16 != f16) return fail(c, BGS_EINVAL, "download: the cloud is in the %s layout", cl->f16 ? "f16" : "f32");
    CU(c, cudaSetDevice(c->device));
    TRY(wait_cloud_steps(c, cl));
    cudaStream_t q = c->stream;
    const uint32_t n = cl->n, m_max = std::min(n, DOWNLOAD_CHUNK);
    const size_t sh_b = f16 ? 96 : 192, so_b = f16 ? 0 : 16;
    const size_t plane_b[4] = {16, sh_b, 16, so_b};          // pos | sh | rot | so, per gaussian
    // (sized once for the largest chunk of either layout: it never grows)
    if (!c->h_bounce) CU(c, cudaMallocHost(&c->h_bounce, 2 * DOWNLOAD_BOUNCE_BYTES));
    const size_t chunk_b = DOWNLOAD_BOUNCE_BYTES;
    StreamScratch staging(q);   // sh | rot | so of one chunk
    CU(c, staging.alloc((size_t)m_max * (sh_b + 16 + so_b)));
    uint8_t* st = static_cast<uint8_t*>(staging.p);
    uint8_t* st_rot = st + (size_t)m_max * sh_b;
    uint8_t* st_so = st_rot + (size_t)m_max * 16;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    struct Events { cudaEvent_t* e; ~Events() { for (int k = 0; k < 2; ++k) if (e[k]) cudaEventDestroy(e[k]); } } ev_guard{ev};
    for (cudaEvent_t& e : ev) CU(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    uint8_t* dst[4] = {reinterpret_cast<uint8_t*>(pos_vis), static_cast<uint8_t*>(sh), static_cast<uint8_t*>(rot), static_cast<uint8_t*>(so)};
    const uint32_t chunks = (n + m_max - 1) / m_max;
    // enqueue chunk i into bounce buffer i & 1
    auto enqueue = [&](uint32_t i) -> bgs_status {
        const uint32_t lo = i * m_max, m = std::min(m_max, n - lo);
        uint8_t* hb = c->h_bounce + (i & 1) * chunk_b;
        launch_unpack(f16, cl->blocks, lo, m, st, st_rot, st_so, q);
        CU(c, cudaGetLastError());
        const uint8_t* src[4] = {reinterpret_cast<const uint8_t*>(cl->pos) + (size_t)lo * 16, st, st_rot, st_so};
        for (int p = 0; p < 4; ++p) {
            if (plane_b[p]) CU(c, cudaMemcpyAsync(hb, src[p], (size_t)m * plane_b[p], cudaMemcpyDeviceToHost, q));
            hb += (size_t)m * plane_b[p];
        }
        CU(c, cudaEventRecord(ev[i & 1], q));
        return BGS_OK;
    };
    TRY(enqueue(0));
    for (uint32_t i = 0; i < chunks; ++i) {
        if (i + 1 < chunks) TRY(enqueue(i + 1));
        CU(c, cudaEventSynchronize(ev[i & 1]));
        const uint32_t lo = i * m_max, m = std::min(m_max, n - lo);
        const uint8_t* hb = c->h_bounce + (i & 1) * chunk_b;
        for (int p = 0; p < 4; ++p) {
            if (plane_b[p]) memcpy(dst[p] + (size_t)lo * plane_b[p], hb, (size_t)m * plane_b[p]);
            hb += (size_t)m * plane_b[p];
        }
    }
    return BGS_OK;
}

bgs_status bgs_cloud_download_f32(bgs_context* c, const bgs_cloud* cl, float* pos_vis, float* sh, float* rot_wxyz, float* scale_opacity) {
    return download_common(c, cl, false, pos_vis, sh, rot_wxyz, scale_opacity);
}

bgs_status bgs_cloud_download_f16(bgs_context* c, const bgs_cloud* cl, float* pos_vis, uint32_t* sh_packed, uint32_t* second_plane) {
    return download_common(c, cl, true, pos_vis, sh_packed, second_plane, nullptr);
}

bgs_status bgs_debug_sorted_entries(bgs_context* c, uint32_t* out) {
    if (!c || !out) return BGS_EINVAL;
    if (!c->have_frame || !c->last.cloud) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    CU(c, cudaSetDevice(c->device));
    const uint32_t n = c->last.cloud->n, n_vis = c->stats.n_visible;
    const uint32_t n_sorted = c->last.sort_all ? n : n_vis;
    std::vector<uint32_t> k(n_sorted), v(n_sorted);
    CU(c, cudaMemcpy(k.data(), c->keys[c->depth_result].p, (size_t)n_sorted * 4, cudaMemcpyDeviceToHost));
    CU(c, cudaMemcpy(v.data(), c->vals[c->depth_result].p, (size_t)n_sorted * 4, cudaMemcpyDeviceToHost));
    if (c->last.by_slot) {   // the sort's payload is the compact slot: map it to the gaussian index
        std::vector<uint32_t> ids(n_sorted);
        CU(c, cudaMemcpy(ids.data(), c->slot_ids.p, (size_t)n_sorted * 4, cudaMemcpyDeviceToHost));
        for (uint32_t i = 0; i < n_sorted; ++i) v[i] = ids[v[i]];
    }
    for (uint32_t i = 0; i < n_sorted; ++i) { out[2 * i] = k[i]; out[2 * i + 1] = v[i]; }
    if (!c->last.sort_all) {
        // culled tail: key = all-ones >> shift, indices ascending (what a stable sort leaves there)
        uint32_t* flags = nullptr;
        CU(c, cudaMalloc(&flags, (size_t)n * 4));
        launch_culled_flags(c->last.cloud->pos, n, c->last.fc, flags, c->stream);
        std::vector<uint32_t> f(n);
        cudaError_t e = cudaMemcpyAsync(f.data(), flags, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        cudaFree(flags);
        if (e != cudaSuccess) return fail(c, BGS_ECUDA, "debug_sorted_entries: %s", cudaGetErrorString(e));
        const uint32_t culled_key = 0xFFFFFFFFu >> c->last.fc.key_shift;
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
    if (c->last.rounds > 1) return fail(c, BGS_NOT_READY, "the last frame was binned in %d rounds: set BGS_FLAG_NO_CHUNKS for the tile hooks", c->last.rounds);
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
    if (c->last.rounds > 1) return fail(c, BGS_NOT_READY, "the last frame was binned in %d rounds: set BGS_FLAG_NO_CHUNKS for the tile hooks", c->last.rounds);
    CU(c, cudaSetDevice(c->device));
    const uint64_t cnt = c->stats.n_pairs < capacity ? c->stats.n_pairs : capacity;
    CU(c, cudaMemcpy(ranks, c->pvals[c->pair_result].p, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    if (c->last.by_slot) {   // pair payload = record index = compact slot: convert to front-to-back rank
        const uint32_t n_vis = c->stats.n_visible;
        std::vector<uint32_t> perm(n_vis), inv(n_vis);
        CU(c, cudaMemcpy(perm.data(), c->vals[c->depth_result].p, (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
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
    CU(c, cudaMemcpy(v.data(), c->vals[c->depth_result].p, (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
    if (c->last.by_slot) {
        ids.resize(n_vis);
        CU(c, cudaMemcpy(ids.data(), c->slot_ids.p, (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
    }
    if (records) {
        std::vector<SplatRec> tmp(n_vis);
        CU(c, cudaMemcpy(tmp.data(), c->recs.p, (size_t)n_vis * sizeof(SplatRec), cudaMemcpyDeviceToHost));
        for (uint32_t r = 0; r < n_vis; ++r) {
            const uint32_t ri = c->last.by_slot ? v[n_vis - 1 - r] : r;   // rank -> record index
            memcpy(records + (size_t)r * 12, &tmp[ri], sizeof(SplatRec));
        }
    }
    if (rank_to_index)
        for (uint32_t r = 0; r < n_vis; ++r) rank_to_index[r] = c->last.by_slot ? ids[v[n_vis - 1 - r]] : v[n_vis - 1 - r];
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
        const void* f = c->frames[k].p;
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
    return c->have_frame ? c->last.target : (c->async_pending ? c->pend.target : nullptr);
}
uint32_t bgs_last_launch_count(const bgs_context* c) { return c ? c->launches : 0; }

}  // extern "C"
