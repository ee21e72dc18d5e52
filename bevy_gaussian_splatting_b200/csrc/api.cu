// api.cu -- the extern "C" boundary of libbgs (include/bgs.h): contexts, the per-view frame (stage orchestration on
// one CUDA stream), parity/debug hooks, stage timing.  The calls on a resident cloud are in cloud.cu.
//
// No PyTorch, no wgpu, no CPU fallback: every stage is a hand-written sm_90a kernel.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <new>
#include <vector>

#include "host.cuh"

namespace bgs {

std::mutex g_registry_mu;
std::vector<bgs_context*> g_contexts;
std::vector<bgs_entity_list*> g_lists;

bgs_status fail(bgs_context* ctx, bgs_status st, const char* fmt, ...) {
    if (ctx) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
        va_end(ap);
    }
    return st;
}

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

// look-back status rows of a sort of up to `capacity` entries: 4 passes x tiles x 256 digits x 8 B, epoch-tagged
// (radix.cu), so they are cleared exactly once -- when allocated -- and never again
bgs_status ensure_status(bgs_context* c, DevBuf<void>& rows, uint32_t& rows_capacity, uint32_t capacity) {
    if (capacity <= rows_capacity) return BGS_OK;
    rows_capacity = 0;
    TRY(rows.grow(c, (size_t)4 * radix_num_tiles(capacity) * 256 * 8, true));
    rows_capacity = capacity;
    return BGS_OK;
}

void detach_listed_cloud(const bgs_cloud* cl) {
    for (bgs_entity_list* l : g_lists) {
        const auto it = l->clouds.find(cl);
        if (it == l->clouds.end()) continue;
        l->clouds.erase(it);
        for (ListEntity& x : l->ent)
            if (x.cloud == cl) { x.cloud = nullptr; ++l->detached; }
    }
}

uint32_t next_epoch(bgs_context* c) {
    if (++c->sort_epoch >= (1u << 30)) {     // (2^30 sorts later) start over from clean rows
        for (DevBuf<void>* s : {&c->status_depth, &c->status_pairs})
            if (s->p) cudaMemsetAsync(s->p, 0, s->bytes, c->stream);
        c->sort_epoch = 1;
    }
    return c->sort_epoch;
}

}  // namespace bgs

namespace {

constexpr uint32_t CHUNK_MAX_TILES = 65536;
// chunked frames (saturation-aware binning): the visible set is binned / sorted / blended in front-to-back rank rounds
// [CHUNK_FRAC[r], CHUNK_FRAC[r + 1]) / 65536; once every tile has saturated the remaining rounds emit nothing
// (x8 schedule: the front of a heavy scene saturates the frame within a few hundred splats)
constexpr uint32_t CHUNK_FRAC[MAX_CHUNKS + 1] = {0, 16, 128, 1024, 8192, 65536};
// CTAs per SM of the cooperative key-gen and binning grids: synchronous frames (latency), queued (BGS_FLAG_ASYNC) frames
constexpr int COOP_CTAS_PER_SM = 4, COOP_CTAS_PER_SM_ASYNC = 1;
// radix-sort CTAs per SM the pair sort of queued frames may use (1: half an SM, two waves)
constexpr int SORT_CTAS_PER_SM_ASYNC = 1;

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
    Layout l;
    const size_t o_ctr = l.add(sizeof(FrameCounters));
    const size_t o_vr = l.add(sizeof(ViewRanges));
    const size_t o_hist = l.add((8 + 4 * MAX_CHUNKS) * 256 * 4);
    // (the queued-frame grids are never larger than the synchronous ones)
    const size_t o_kgc = l.add((size_t)c->kg_grid * 4);
    const size_t o_binc = l.add((size_t)c->bin_grid * 3 * 4);
    // chunked frames (only for <= CHUNK_MAX_TILES tiles) use one ranges array per round + a done byte per tile; an
    // arena sized by a larger frame must still hold them for a later, smaller (chunkable) frame
    const size_t chunk_tiles = tiles <= CHUNK_MAX_TILES ? tiles : CHUNK_MAX_TILES;
    const size_t range_entries = chunk_tiles * MAX_CHUNKS > tiles ? chunk_tiles * MAX_CHUNKS : tiles;
    const size_t o_rng = l.add(range_entries * 8);
    const size_t o_done = l.add(chunk_tiles);
    TRY(c->arena.grow(c, l.padded(), false));
    c->ctr = reinterpret_cast<FrameCounters*>(c->arena.p + o_ctr);
    c->view_ranges = reinterpret_cast<ViewRanges*>(c->arena.p + o_vr);
    c->hist = reinterpret_cast<uint32_t*>(c->arena.p + o_hist);
    c->kg_block_cnt = reinterpret_cast<uint32_t*>(c->arena.p + o_kgc);
    c->bin_block_cnt = reinterpret_cast<uint32_t*>(c->arena.p + o_binc);
    c->ranges = reinterpret_cast<uint2*>(c->arena.p + o_rng);
    c->tile_done = c->arena.p + o_done;
    c->arena_tiles = tiles;
    return BGS_OK;
}

size_t format_bpp(uint32_t f) { return f == BGS_FORMAT_RGBA32F ? 16 : (f == BGS_FORMAT_RGBA16F ? 8 : 4); }

// Every choice a frame's launches depend on beyond the frame itself: made from the settings, the previous frame's
// counts (the hints) and the context's grids and capacities.  plan_frame makes no CUDA call and changes nothing.
struct FramePlan {
    int raster_mode;        // 0 = quad-uv falloff (USE_OBB, 3DGS and 2DGS), 1 = 3DGS conic (USE_AABB), 2 = 2DGS ray-splat (USE_AABB)
    int rounds;             // binning rounds: 1, or MAX_CHUNKS on a chunked frame
    bool large_fp;          // blend variant for large footprints (results are identical)
    bool box;               // the bounding-box overlay (BGS_FLAG_VISUALIZE_BOUNDING_BOX): one round, raster_body's blend
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
    p.raster_mode = !st->aabb ? 0 : (st->gaussian_mode == BGS_GAUSSIAN_2D ? 2 : 1);   // (4D records are 3DGS conics)
    // saturation-aware chunking: frames whose splats cover many tiles each (last frame: >= 32 pairs per visible splat
    // and >= 2^24 pairs: below that, one round is cheaper than the extra launches) run binning / tile sort /
    // blend in front-to-back rank rounds; the rounds after every tile has saturated emit nothing.
    // Quad-uv records only, and not on overlay frames (like aux frames); BGS_FLAG_CHUNKS / _NO_CHUNKS force it.
    p.box = (st->flags & BGS_FLAG_VISUALIZE_BOUNDING_BOX) != 0;
    bool chunked = p.raster_mode == 0 && !want_aux && !p.box && num_tiles <= CHUNK_MAX_TILES && !(st->flags & BGS_FLAG_NO_CHUNKS);
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

// What a frame writes, and where: each of v views' colour frame rgba[i] and, on aux frames, its depth and normal frames
// depth[i] and normal[i], and on pick frames (bgs_render_entities_pick) the pick frame `pick` (else NULL), in `format`, in
// device memory (`device`) or host memory.  A single-view frame is view 0.  A shutter frame (bgs_render_shutter): the v
// views are its samples, whose blends go to the context's sub-frames, and rgba[0] is its one frame.
struct Targets {
    uint32_t format;
    int device;
    uint32_t v;
    bool aux;
    void* const* rgba;
    void* const* depth;
    void* const* normal;
    void* pick;
    bool shutter = false;
};
// a single-view frame's colour frame alone
Targets colour_target(void* const* rgba, uint32_t format, int device) {
    return {format, device, 1, false, rgba, nullptr, nullptr, nullptr};
}

// Where a frame's pixels go.
struct FrameOut {
    uint32_t raster_format = 0;         // output mode of the blend kernels: format | mode << 8 (raster.cu)
    int slot = -1;                      // a queued frame in the library's own frames: which of the two (else -1)
    // view i's bytes (of one frame), its device targets (the caller's frames or the library's), and the host frames they
    // are copied to (host targets; else NULL); the depth and normal ones on aux frames
    uint32_t v = 1;
    size_t bytes[MAX_VIEWS] = {};
    void* rgba[MAX_VIEWS] = {};
    void* depth[MAX_VIEWS] = {};
    void* normal[MAX_VIEWS] = {};
    void* host_rgba[MAX_VIEWS] = {};
    void* host_depth[MAX_VIEWS] = {};
    void* host_normal[MAX_VIEWS] = {};
    // a pick frame (bgs_render_entities_pick): its device records, the host target they are copied to (else NULL)
    uint4* pick = nullptr;
    void* host_pick = nullptr;
};

// A frame's targets, view i W[i] x H[i] pixels: the caller's device frames, or the library's own (grown on demand), which
// hold every view's frame one after another (aux frames: frame_aux[0] every view's depth frame, frame_aux[1] every normal
// frame) and are copied to the caller's host frames
bgs_status frame_out(bgs_context* c, const bgs_settings* st, const Targets& t, const int* W, const int* H, FrameOut* o) {
    const bool blend_over = (st->flags & BGS_FLAG_BLEND_OVER_TARGET) != 0;
    o->raster_format = t.format | ((blend_over ? 2u : ((st->flags & BGS_FLAG_PREMULTIPLIED_OUT) ? 1u : 0u)) << 8);
    const size_t bpp = format_bpp(t.format);
    o->v = t.v;
    size_t total = 0;
    for (uint32_t i = 0; i < t.v; ++i) total += o->bytes[i] = (size_t)W[i] * H[i] * bpp;
    // device targets are written with pixel-sized vector stores (and read so in blend-over mode): each must be aligned to
    // one pixel, 4 / 8 / 16 bytes
    if (t.device)
        for (uint32_t i = 0; i < t.v; ++i)
            for (const void* p : {t.rgba[i], t.aux ? t.depth[i] : nullptr, t.aux ? t.normal[i] : nullptr})
                if (reinterpret_cast<uintptr_t>(p) % bpp != 0)
                    return fail(c, BGS_EINVAL, "render: device target %p is not aligned to its %zu-byte pixels", p, bpp);
    if (t.device && t.rgba[0]) {
        for (uint32_t i = 0; i < t.v; ++i) o->rgba[i] = t.rgba[i];
    } else {
        for (int k = 0; k < 2; ++k) {
            if (total <= c->frames[k].bytes) continue;
            TRY(c->frames[k].grow(c, total, true));      // (BGS_FLAG_BLEND_OVER_TARGET reads the target)
            c->copy_pending[k] = false;
        }
        // async frames rendered into the library's own buffers alternate two device frames, so whatever consumes
        // frame k off the render stream (the D2H copy, the NCCL gather: both on the copy/comm stream) overlaps frame k+1
        // (blend-over, queued or not, keeps blending into the frame the previous call produced; synchronous calls that do
        // not blend over use frame 0)
        int k = 0;
        if (blend_over) k = c->frame_last;
        else if (st->flags & BGS_FLAG_ASYNC) { k = c->frame_toggle; c->frame_toggle ^= 1; }
        c->frame_last = k;
        if (st->flags & BGS_FLAG_ASYNC) o->slot = k;
        size_t at = 0;
        for (uint32_t i = 0; i < t.v; at += o->bytes[i++]) {
            o->rgba[i] = static_cast<char*>(c->frames[k].p) + at;
            o->host_rgba[i] = t.rgba[i];
        }
    }
    if (t.aux && t.device) {
        for (uint32_t i = 0; i < t.v; ++i) { o->depth[i] = t.depth[i]; o->normal[i] = t.normal[i]; }
    } else if (t.aux) {
        for (int k = 0; k < 2; ++k) TRY(c->frame_aux[k].grow(c, total, true));
        size_t at = 0;
        for (uint32_t i = 0; i < t.v; at += o->bytes[i++]) {
            o->depth[i] = static_cast<char*>(c->frame_aux[0].p) + at;
            o->normal[i] = static_cast<char*>(c->frame_aux[1].p) + at;
            o->host_depth[i] = t.depth[i];
            o->host_normal[i] = t.normal[i];
        }
    }
    if (t.pick && t.device) {
        o->pick = static_cast<uint4*>(t.pick);
    } else if (t.pick) {
        TRY(c->pick_frame.grow(c, (size_t)W[0] * H[0] * sizeof(bgs_pick), false));
        o->pick = c->pick_frame.p;
        o->host_pick = t.pick;
    }
    return BGS_OK;
}

}  // namespace

namespace bgs {

FrameConsts frame_consts(const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                                const bgs_settings* st, bool want_aux) {
    return make_frame_consts(*view, *uni, st->radix_sort_depth_bits, st->gaussian_mode, st->rasterize_mode, st->aabb,
                             st->opacity_adaptive_radius, st->draw_mode, cloud->n,
                             cloud->layout == CloudLayout::F16Cov ? 1u : 0u, want_aux ? 1u : 0u);
}

}  // namespace bgs

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
    if (e == cudaSuccess) e = cudaMallocHost(&c->h_sticky, 4);
    if (e == cudaSuccess) e = cudaMallocHost(&c->h_word, 4);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_sticky, 16);
    if (e == cudaSuccess) e = cudaMemset(c->d_sticky, 0, 16);
    if (e == cudaSuccess) e = cudaMalloc(&c->cutoff_tab, 65536 * sizeof(float));
    if (e == cudaSuccess) { launch_cutoff_table(c->cutoff_tab, c->stream); e = cudaStreamSynchronize(c->stream); }
    if (e == cudaSuccess) *c->h_sticky = 0;
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
        c->kg_scene_per_sm = (uint32_t)keygen_scene_blocks_per_sm();
        c->kg_many_per_sm = (uint32_t)keygen_many_blocks_per_sm();
        if (c->kg_grid == 0 || c->bin_grid == 0 || c->rs_per_sm == 0 || c->kg_scene_per_sm == 0 || c->kg_many_per_sm == 0) coop = 0;
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
    // its lists refuse every later call; their device arrays go once the context's streams are drained
    std::vector<std::shared_ptr<ListTable>> tables;
    std::vector<void*> uploads;
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);
        g_contexts.erase(std::remove(g_contexts.begin(), g_contexts.end(), c), g_contexts.end());
        for (bgs_entity_list* l : g_lists)
            if (l->ctx == c) {
                tables.push_back(std::move(l->cur));
                tables.push_back(std::move(l->spare));
                uploads.push_back(l->upload.p);
                l->upload.p = nullptr;
                l->upload.bytes = 0;
                l->ctx = nullptr;
            }
    }
    cudaSetDevice(c->device);
    c->each_stream([](cudaStream_t& s, int) { if (s) cudaStreamSynchronize(s); });
    tables.clear();
    for (void* u : uploads) cudaFree(u);
    c->each_event([](cudaEvent_t& ev, bool) { if (ev) cudaEventDestroy(ev); });
    c->each_stream([](cudaStream_t& s, int) { if (s) cudaStreamDestroy(s); });
    if (c->h_ctr) cudaFreeHost(c->h_ctr);
    if (c->h_sticky) cudaFreeHost(c->h_sticky);
    if (c->h_word) cudaFreeHost(c->h_word);
    if (c->h_bounce) cudaFreeHost(c->h_bounce);
    for (auto& m : c->many)
        if (m.host) cudaFreeHost(m.host);
    cudaFree(c->d_sticky);
    cudaFree(c->cutoff_tab);
    delete c;   // (releases every DevBuf)
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
    if (!c->async_pending && !c->step_pending && !c->reads_pending.load(std::memory_order_relaxed)) return BGS_OK;
    CU(c, cudaSetDevice(c->device));
    c->step_pending = false;
    if (!c->async_pending) {   // only particle steps or interpolations were queued: no frame to account for
        CU(c, cudaStreamSynchronize(c->stream));
        c->reads_pending.store(false, std::memory_order_relaxed);
        CU(c, cudaGetLastError());
        return BGS_OK;
    }
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaStreamSynchronize(c->stream_copy));
    c->reads_pending.store(false, std::memory_order_relaxed);
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

// check_render's refusals of the frame's format and sort bits
static bgs_status check_frame_bits(bgs_context* c, const bgs_settings* st, uint32_t out_format) {
    if (out_format > BGS_FORMAT_RGBA32F) return fail(c, BGS_EINVAL, "render: unknown out_format %u", out_format);
    if (st->radix_sort_depth_bits != 16 && st->radix_sort_depth_bits != 24 && st->radix_sort_depth_bits != 32)
        return fail(c, BGS_EINVAL, "render: radix_sort_depth_bits must be 16, 24 or 32");
    return BGS_OK;
}

// ... of an OpticalFlow frame's extras
static bgs_status check_flow_extras(bgs_context* c, const bgs_render_extras* ex) {
    if (!ex) return fail(c, BGS_EINVAL, "render: OpticalFlow needs the previous view (bgs_render_ex extras)");
    if (!(std::isfinite(ex->delta_time) && ex->delta_time > 0.0f))
        return fail(c, BGS_EINVAL, "render: OpticalFlow delta_time %g is not finite and > 0", (double)ex->delta_time);
    for (int i = 0; i < 16; ++i)
        if (!std::isfinite(ex->previous_clip_from_world[i]))
            return fail(c, BGS_EINVAL, "render: previous_clip_from_world[%d] is not finite", i);
    return BGS_OK;
}

// ... of the view
static bgs_status check_viewport(bgs_context* c, const bgs_view* view) {
    const int W = (int)view->viewport[2], H = (int)view->viewport[3];
    if (W <= 0 || H <= 0 || W > 65535 || H > 65535) return fail(c, BGS_EINVAL, "render: viewport %dx%d out of range", W, H);
    return BGS_OK;
}

// ... of the cloud's layout and the settings (ex: the extras as the call reads them, NULL for none), which depend on
// nothing else but the OpticalFlow extras, checked only with `flow` (bgs_entity_list checks an entity's settings at the
// edit, and the frame's extras when it renders)
static bgs_status check_settings(bgs_context* c, const bgs_cloud* cloud, const bgs_settings* st, const bgs_render_extras* ex,
                                 bool want_aux, bool temporal, bool flow) {
    if (temporal) {
        if (!is_4d(cloud->layout)) return fail(c, BGS_EINVAL, "render_4d: the cloud is not a Gaussian4d cloud (bgs_cloud_upload_4d)");
        if (st->gaussian_mode != BGS_GAUSSIAN_4D)
            return fail(c, BGS_EINVAL, "render_4d: gaussian_mode %u is not BGS_GAUSSIAN_4D", st->gaussian_mode);
        if (st->rasterize_mode > BGS_RASTERIZE_VELOCITY || st->rasterize_mode == BGS_RASTERIZE_NORMAL)
            return fail(c, BGS_EINVAL, "render_4d: rasterize_mode %u not supported (Normal has no 4D rotation)", st->rasterize_mode);
    } else {
        if (is_4d(cloud->layout)) return fail(c, BGS_EINVAL, "render: a Gaussian4d cloud renders through bgs_render_4d");
        if (st->gaussian_mode != BGS_GAUSSIAN_3D && st->gaussian_mode != BGS_GAUSSIAN_2D)
            return fail(c, BGS_EINVAL, "render: gaussian_mode %u not supported here (Gaussian4d: bgs_render_4d)", st->gaussian_mode);
        if (st->rasterize_mode > BGS_RASTERIZE_OPTICAL_FLOW)
            return fail(c, BGS_EINVAL, "render: rasterize_mode %u not supported here (Velocity: bgs_render_4d)", st->rasterize_mode);
    }
    if (st->rasterize_mode >= BGS_RASTERIZE_CLASSIFICATION && want_aux)
        return fail(c, BGS_EINVAL, "render_aux: Classification and OpticalFlow frames take extras: use bgs_render_ex");
    if (st->rasterize_mode == BGS_RASTERIZE_CLASSIFICATION && ex && ex->num_classes == 0)
        return fail(c, BGS_EINVAL, "render: Classification with num_classes = 0");
    if (flow && st->rasterize_mode == BGS_RASTERIZE_OPTICAL_FLOW) TRY(check_flow_extras(c, ex));
    if (st->draw_mode > BGS_DRAW_HIGHLIGHT_SELECTED) return fail(c, BGS_EINVAL, "render: bad draw_mode");
    if (cloud->layout == CloudLayout::F16Cov && (st->gaussian_mode != BGS_GAUSSIAN_3D || st->rasterize_mode == BGS_RASTERIZE_NORMAL || want_aux))
        return fail(c, BGS_EINVAL, "render: a precomputed-covariance cloud has no rotation / scale: Gaussian3d with Color, Depth or Position only");
    return BGS_OK;
}

static bgs_status check_render(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                               const bgs_settings* st, const bgs_render_extras* ex, uint32_t out_format, bool want_aux,
                               bool temporal, bool set_device = true) {
    // not-ready inputs map to the reference's silent skip-frame (radix.rs:645-658, mod.rs:1533-1539)
    if (!cloud || !view || !uni || !st) return fail(c, BGS_NOT_READY, "render: cloud/view/uniform/settings not ready");
    // (contexts of one GPU may share clouds; a scene's entities after its first only check the device, which the first
    // made current)
    if (set_device) TRY(enter_call(c, "render", cloud->device));
    else if (cloud->device != c->device) return fail(c, BGS_EINVAL, "render: cloud lives on another device");
    TRY(check_frame_bits(c, st, out_format));
    TRY(check_settings(c, cloud, st, ex, want_aux, temporal, true));
    return check_viewport(c, view);
}


// Enqueues one attempt at a frame: every launch of the plan, the counters' read-back and the copy-out.  A scene frame
// (render_entities_impl) runs key-gen, the depth range, the projection and the splat depths over its segment table; `cloud`
// is then its first cloud and fc its first segment's.  sub_frames non-null (a shutter frame, with views): the views blend
// stores each view's raw (C, T) at views->out[i], slices of sub_frames, and the resolve writes the frame o.rgba[0].
static bgs_status enqueue_frame(bgs_context* c, const bgs_cloud* cloud, const FrameConsts& fc, const ModeConsts* modes,
                                const TemporalConsts* tc, const FramePlan& p, const FrameOut& o, const bgs_scene_depth* zd,
                                const std::shared_ptr<const SceneFacts>& scene, const ViewTable* views,
                                const float4* sub_frames) {
    const uint32_t n = scene ? scene->tab.n_total : cloud->n;
    // (a views frame: every view's tiles, one global tile id space)
    const uint32_t num_tiles = views ? views->tile0[views->v] : (uint32_t)fc.tiles_x * (uint32_t)fc.tiles_y;
    cudaStream_t q = c->stream;
    uint32_t launches = 0;
    if (scene) {
        for (const bgs_cloud* cl : scene->distinct) TRY(before_cloud_read(c, cl));
    } else {
        TRY(before_cloud_read(c, cloud));
    }
    const bool many = scene && scene->many;   // (bgs_render_entities_many: the segment table in device memory)
    const SceneTableDev* dt = many ? &scene->dtab : nullptr;
    if (many && scene->list_tab) {   // (bgs_render_entity_list: the segments from the list's records and the view)
        const ListTable& lt = *scene->list_tab;
        CU(c, launch_entity_list_expand(lt.a.recs, lt.a.offset, dt->k, scene->list_view, scene->list_depth_bits, dt->n_total,
                                        lt.seg, q));
        ++launches;
    } else if (many) {
        CU(c, cudaMemcpyAsync(c->many[scene->slot].dev.p, scene->h_tab, scene->tab_bytes, cudaMemcpyHostToDevice, q));
    }
    CU(c, cudaMemsetAsync(c->arena.p, 0, c->arena.bytes, q));   // counters, histograms, ranges: ~0.4 MB
    CU(c, cudaEventRecord(c->ev[0], q));
    // ---- stage 1: key-gen (+ stable compaction of the visible set)
    // compact mode: keys[0][slot], slot_ids[slot] = gaussian index, vals[0][slot] = slot (sort payload)
    // SORT_ALL    : keys[0][i], vals[0][i] = i (payload is the gaussian index itself)
    if (scene) {   // (scenes are compact frames)
        // key-gen gathers the culled ends for the Depth range when segment 0 is in Depth mode: when only some other
        // entity is, it reads a copy of the table whose segment 0 is
        const bool depth0 = p.depth_range && scene->tab.seg[0].fc.rasterize_mode != BGS_RASTERIZE_DEPTH;
        if (many) {   // (the frame-wide values are an argument of their own)
            FrameConsts f0 = scene->tab.seg[0].fc;
            if (depth0) f0.rasterize_mode = BGS_RASTERIZE_DEPTH;
            CU(c, launch_keygen_many(*dt, f0, c->keys[1].p, c->keys[0].p, c->slot_ids.p, c->vals[0].p, c->kg_block_cnt, c->ctr,
                                     c->hist, p.depth_passes, std::min(p.kg_grid, (uint32_t)c->sm_count * c->kg_many_per_sm), q));
        } else {
            SceneTable kt;
            if (depth0) {
                kt = scene->tab;
                kt.seg[0].fc.rasterize_mode = BGS_RASTERIZE_DEPTH;
            }
            CU(c, launch_keygen_scene(depth0 ? kt : scene->tab, c->keys[1].p, c->keys[0].p, c->slot_ids.p, c->vals[0].p,
                                      c->kg_block_cnt, c->ctr, c->hist, p.depth_passes,
                                      std::min(p.kg_grid, (uint32_t)c->sm_count * c->kg_scene_per_sm), q));
        }
    } else if (p.by_slot) {
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
    // (a views aux frame: each view's range from its own entries, which its projection reads)
    const bool view_ranges = views && fc.aux;
    if (p.depth_range) {
        if (view_ranges) launch_depth_range_views(scene->tab, views->v, views->n_view, c->vals[cur].p, c->slot_ids.p, c->ctr,
                                                  c->view_ranges, p.n_hint, c->sm_count, q);
        else if (many) launch_depth_range_many(*dt, c->vals[cur].p, c->slot_ids.p, c->ctr, q);
        else if (scene) launch_depth_range_scene(scene->tab, c->vals[cur].p, c->slot_ids.p, c->ctr, q);
        else launch_depth_range(cloud->pos, n, c->vals[cur].p, p.by_slot ? c->slot_ids.p : nullptr, c->ctr, fc, q);
        ++launches;
    }
    CU(c, cudaEventRecord(c->ev_p0, ps));
    bool scene_3d = false;   // a scene lists a non-4D cloud (whose splat depths splat_depth_scene writes)
    if (scene) {   // one launch per projection group: each segment with its own settings and num_classes
        for (size_t i = 0; i < scene->groups.size(); ++i) {
            const uint32_t g = scene->groups[i];
            if (many) {
                launch_project_many(*dt, g, scene->need_sh[i] != 0, *modes, c->slot_ids.p, c->ctr, c->recs.p,
                                    (p.raster_mode == 2 || p.raster_mode == 4) ? c->extra.p : nullptr,
                                    zd || o.pick ? c->splat_depth.p : nullptr, p.n_hint, c->sm_count, c->cutoff_tab, ps);
                scene_3d = scene_3d || g != PROJECT_GROUP_4D;
            } else if (g == PROJECT_GROUP_4D) {   // (also writes the 4D segments' splat depths, from the moved positions)
                launch_project_4d_scene(scene->tab, scene->times, scene->classes, *modes, c->slot_ids.p, c->ctr, c->recs.p,
                                        zd || o.pick ? c->splat_depth.p : nullptr, p.n_hint, c->sm_count, ps);
            } else {
                launch_project_scene(scene->tab, g, scene->need_sh[i] != 0, scene->classes, *modes, c->slot_ids.p, c->ctr,
                                     c->recs.p, (p.raster_mode == 2 || p.raster_mode == 4) ? c->extra.p : nullptr, p.n_hint,
                                     c->sm_count, c->cutoff_tab, fc.aux ? c->aux.p : nullptr, ps,
                                     view_ranges ? c->view_ranges : nullptr, view_ranges ? scene->tab.k / views->v : 0u);
                scene_3d = true;
            }
            ++launches;
        }
    } else if (tc) {   // Gaussian4d: the projection also writes the depth-tested frame's splat depths, from the moved positions
        launch_project_4d(cloud->blocks, p.by_slot ? c->slot_ids.p : c->vals[cur].p, p.by_slot ? 1 : 0, c->ctr, fc,
                          modes ? *modes : ModeConsts{}, *tc, c->recs.p, zd ? c->splat_depth.p : nullptr, p.n_hint, c->sm_count, ps);
    } else {
        launch_project(cloud->layout, cloud->sh_degree, cloud->blocks, p.by_slot ? c->slot_ids.p : c->vals[cur].p,
                       p.by_slot ? 1 : 0, c->ctr, fc, c->recs.p, p.raster_mode == 2 ? c->extra.p : nullptr, p.n_hint, c->sm_count, c->cutoff_tab,
                       fc.aux ? c->aux.p : nullptr, modes, ps);
    }
    if (!scene) ++launches;
    CU(c, cudaEventRecord(c->ev_p1, ps));
    // depth-tested and pick frames: the splat depths, indexed like the records (the projection's index list)
    if ((zd || o.pick) && scene_3d) {
        if (many) launch_splat_depth_many(*dt, c->slot_ids.p, c->ctr, c->splat_depth.p, p.n_hint, c->sm_count, ps);
        else launch_splat_depth_scene(scene->tab, c->slot_ids.p, c->ctr, c->splat_depth.p, p.n_hint, c->sm_count, ps);
        ++launches;
    } else if (zd && !tc && !scene) {
        launch_splat_depth(cloud->pos, p.by_slot ? c->slot_ids.p : c->vals[cur].p, p.by_slot ? 1 : 0, c->ctr, fc,
                           c->splat_depth.p, p.n_hint, c->sm_count, ps);
        ++launches;
    }
    // the blend's inputs (each round: its pair list and ranges) and targets
    BlendArgs b;
    b.mode = p.raster_mode;
    b.box = p.box;
    b.large_footprints = p.large_fp;
    b.recs = c->recs.p;
    b.extra = c->extra.p;
    b.W = fc.Wi; b.H = fc.Hi; b.tiles_x = fc.tiles_x; b.tiles_y = fc.tiles_y;
    b.out = o.rgba[0];
    b.format = o.raster_format;
    b.aux = fc.aux ? c->aux.p : nullptr;
    b.out_depth = o.depth[0];
    b.out_normal = o.normal[0];
    b.truncated = &c->ctr->truncated;
    if (zd || o.pick) b.splat_d = c->splat_depth.p;
    if (zd) { b.scene = zd->depth; b.pitch = (size_t)zd->pitch_bytes; }
    b.kinds = c->kinds.p;
    b.views = views;
    b.raw = sub_frames != nullptr;
    PickArgs pk = {};
    PickArgsDev pkd = {};
    if (o.pick && many) {
        pkd = PickArgsDev{o.pick, c->slot_ids.p, *dt};
        b.pick_dev = &pkd;
    } else if (o.pick) {
        pk = PickArgs{o.pick, c->slot_ids.p, scene->kinds};
        b.pick = &pk;
    }
    if (p.overlap) {
        CU(c, cudaEventRecord(c->ev_join, c->stream2));
        CU(c, cudaStreamWaitEvent(q, c->ev_join, 0));
    }
    CU(c, cudaEventRecord(c->ev[3], q));
    if (p.raster_mode >= 3) {   // a mixed-geometry frame: each record's blend kind, for the blend
        if (many) launch_segment_kinds_many(*dt, c->slot_ids.p, c->ctr, c->kinds.p, p.n_hint, c->sm_count, q);
        else launch_segment_kinds(scene->kinds, c->slot_ids.p, c->ctr, c->kinds.p, p.n_hint, c->sm_count, q);
        ++launches;
    }
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
        if (views)   // (one round)
            CU(c, launch_bin_emit_views(c->recs.p, c->vals[cur].p, c->ctr, cc, num_tiles, c->bin_block_cnt, c->cap_pairs,
                                        c->pkeys[0].p, c->pvals[0].p, c->keys[cur ^ 1].p, c->vals[cur ^ 1].p, c->cap_n,
                                        p.bin_grid, c->d_sticky, c->slot_ids.p, *views, c->sm_count, q));
        else CU(c, launch_bin_emit_coop(c->recs.p, p.by_slot ? c->vals[cur].p : nullptr, c->ctr, cc, fa, fb, num_tiles,
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
        b.tile_entries = c->pvals[pcur].p;
        b.ranges = rng;
        if (r + 1 == p.rounds) {
            // (chunked frames: the earlier rounds' blends are accounted to stage 4)
            CU(c, cudaEventRecord(c->ev[4], q));
            if (o.slot >= 0 && c->copy_pending[o.slot]) CU(c, cudaStreamWaitEvent(q, c->ev_copied[o.slot], 0));   // target free again
        }
        if (p.rounds == 1) {
            // the blend runs on the LOW-priority stream; the render stream resumes once it is done
            CU(c, cudaEventRecord(c->ev_front, q));
            CU(c, cudaStreamWaitEvent(c->stream_r, c->ev_front, 0));
            launch_raster(b, c->stream_r);
            CU(c, cudaEventRecord(c->ev_rdone, c->stream_r));
            CU(c, cudaStreamWaitEvent(q, c->ev_rdone, 0));
        } else
            launch_raster_round(b, c->state.p, c->tile_done, &c->ctr->tiles_done, r == 0, r + 1 == p.rounds, q);
        ++launches;
    }
    if (sub_frames) {   // (after the blend, which the render stream has joined)
        launch_shutter_resolve(sub_frames, views->v, (uint32_t)fc.Wi * (uint32_t)fc.Hi, o.rgba[0], o.raster_format,
                               &c->ctr->truncated, q);
        ++launches;
    }
    c->pair_result = pcur;
    CU(c, cudaEventRecord(c->ev[5], q));
    CU(c, cudaEventRecord(c->ev_done, q));
    if (many && !scene->list_tab) {   // (the table's last reader is the blend, which the render stream has joined)
        CU(c, cudaEventRecord(c->many[scene->slot].ev, q));
        c->many[scene->slot].used = true;
        c->many_last = scene->slot;
    }
    CU(c, cudaMemcpyAsync(c->h_ctr, c->ctr, sizeof(FrameCounters), cudaMemcpyDeviceToHost, q));
    CU(c, cudaMemcpyAsync(c->h_sticky, c->d_sticky, 4, cudaMemcpyDeviceToHost, q));
    if (o.slot >= 0) CU(c, cudaEventRecord(c->ev_raster[o.slot], q));
    // host targets: each view's frames, then the pick frame, copied out; a queued frame's on the copy stream, after its blend
    if (o.host_rgba[0]) {
        cudaStream_t s = q;
        if (o.slot >= 0) {
            CU(c, cudaStreamWaitEvent(c->stream_copy, c->ev_raster[o.slot], 0));
            s = c->stream_copy;
        }
        for (uint32_t i = 0; i < o.v; ++i) {
            CU(c, cudaMemcpyAsync(o.host_rgba[i], o.rgba[i], o.bytes[i], cudaMemcpyDeviceToHost, s));
            if (o.host_depth[i]) {
                CU(c, cudaMemcpyAsync(o.host_depth[i], o.depth[i], o.bytes[i], cudaMemcpyDeviceToHost, s));
                CU(c, cudaMemcpyAsync(o.host_normal[i], o.normal[i], o.bytes[i], cudaMemcpyDeviceToHost, s));
            }
        }
        if (o.host_pick)
            CU(c, cudaMemcpyAsync(o.host_pick, o.pick, (size_t)fc.Wi * fc.Hi * sizeof(bgs_pick), cudaMemcpyDeviceToHost, s));
        if (o.slot >= 0) {
            CU(c, cudaEventRecord(c->ev_copied[o.slot], c->stream_copy));
            c->copy_pending[o.slot] = true;
        }
    }
    c->pend = {cloud, n, fc, !p.by_slot, p.by_slot, p.rounds, views ? (int)num_tiles : fc.tiles_x, views ? 1 : fc.tiles_y, fc.Wi,
               fc.Hi, o.rgba[0], zd != nullptr || o.pick != nullptr, scene};
    c->launches = launches;
    return BGS_OK;
}

// bgs_render_depth_test's refusals (include/bgs.h): the buffer must be 4-byte aligned device memory of the context's GPU
// with a pitch that holds a row of the viewport
static bgs_status check_scene_depth(bgs_context* c, const bgs_scene_depth* zd, const bgs_view* view) {
    const uint64_t W = (uint64_t)view->viewport[2];
    if (!zd->depth) return fail(c, BGS_EINVAL, "render_depth_test: depth->depth is NULL");
    if (zd->pitch_bytes % 4 != 0 || zd->pitch_bytes < 4 * W)
        return fail(c, BGS_EINVAL, "render_depth_test: pitch %llu is not a multiple of 4 of at least 4 w = %llu",
                    (unsigned long long)zd->pitch_bytes, (unsigned long long)(4 * W));
    if (reinterpret_cast<uintptr_t>(zd->depth) % 4 != 0)
        return fail(c, BGS_EINVAL, "render_depth_test: depth buffer %p is not 4-byte aligned", (const void*)zd->depth);
    cudaPointerAttributes a = {};
    const cudaError_t e = cudaPointerGetAttributes(&a, zd->depth);
    if (e != cudaSuccess) cudaGetLastError();   // (an unknown pointer: clear the error, refuse below)
    if (e != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != c->device)
        return fail(c, BGS_EINVAL, "render_depth_test: depth buffer %p is not device memory of device %d", (const void*)zd->depth,
                    c->device);
    return BGS_OK;
}

static bgs_status render_impl(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                              const bgs_settings* st, const bgs_render_extras* ex, const Targets& t, const bgs_scene_depth* zd,
                              const TemporalConsts* tc, const std::shared_ptr<const SceneFacts>& scene) {
    if (!c) return BGS_EINVAL;
    if (!scene) TRY(check_render(c, cloud, view, uni, st, ex, t.format, t.aux, tc != nullptr));   // (scenes: per cloud, before)
    if (zd) TRY(check_scene_depth(c, zd, view));
    if (c->async_pending && !(st->flags & BGS_FLAG_ASYNC)) {
        // a synchronous render after queued frames completes them first; their failure (including an overflowed
        // pair list = BGS_NOT_READY) is the caller's to see, so this frame is not rendered on top of it
        TRY(bgs_sync(c));
    }
    const FrameConsts fc = scene ? scene->tab.seg[0].fc : frame_consts(cloud, view, uni, st, t.aux);
    // Classification / OpticalFlow, and every scene frame: the projection takes the extras (NULL extras: num_classes = 1)
    ModeConsts mc = {};
    mc.num_classes = ex ? ex->num_classes : 1u;
    if (ex) { memcpy(mc.prev_clip_from_world, ex->previous_clip_from_world, 64); mc.delta_time = ex->delta_time; }
    const ModeConsts* modes = st->rasterize_mode >= BGS_RASTERIZE_CLASSIFICATION || scene ? &mc : nullptr;
    // a views frame (scene->views.v > 1): every view's tiles and targets
    const bool views = scene && scene->views.v > 1;
    const uint32_t n = scene ? scene->tab.n_total : cloud->n;
    const uint32_t num_tiles = views ? scene->views.tile0[scene->views.v] : (uint32_t)fc.tiles_x * (uint32_t)fc.tiles_y;
    TRY(ensure_cloud_scratch(c, n));
    if (c->cap_pairs == 0) TRY(ensure_pair_scratch(c, std::max(n, 1u << 20)));   // first guess; grows on demand
    FrameOut o;
    Targets to = t;
    if (t.shutter) to.v = 1;   // (one frame, of view 0's size, which every sample has)
    TRY(frame_out(c, st, to, views ? scene->views.W : &fc.Wi, views ? scene->views.H : &fc.Hi, &o));
    // a shutter frame: sample i's blend into its W x H slice of the sub-frames
    const size_t wh = (size_t)fc.Wi * fc.Hi;
    if (t.shutter) TRY(c->sub_frames.grow(c, t.v * wh * sizeof(float4), false));
    ViewTable vt = {};
    if (views) {
        vt = scene->views;
        for (uint32_t i = 0; i < vt.v; ++i) {
            vt.out[i] = t.shutter ? static_cast<void*>(c->sub_frames.p + i * wh) : o.rgba[i];
            vt.out_depth[i] = o.depth[i];
            vt.out_normal[i] = o.normal[i];
        }
    }
    for (int attempt = 0; attempt < 4; ++attempt) {
        FramePlan p = plan_frame(c, st, t.aux, num_tiles, n);   // (each attempt: the pair hints read cap_pairs)
        if (scene) {   // (st plans it as an aabb frame or an overlay one: one round)
            p.raster_mode = scene->raster_mode;
            p.box = scene->box;
        }
        if (p.raster_mode == 2 || p.raster_mode == 4) TRY(c->extra.grow(c, (size_t)c->cap_n * 64, false));
        if (p.raster_mode >= 3) TRY(c->kinds.grow(c, (size_t)c->cap_n, false));
        if (t.aux) TRY(c->aux.grow(c, (size_t)c->cap_n * 32, false));
        if (zd || o.pick) TRY(c->splat_depth.grow(c, (size_t)c->cap_n * 4, false));
        if (p.rounds > 1) TRY(c->state.grow(c, (size_t)num_tiles * 256 * sizeof(float4), false));
        TRY(ensure_arena(c, num_tiles));
        TRY(ensure_status(c, c->status_depth, c->status_n, n));
        TRY(ensure_status(c, c->status_pairs, c->status_np, c->cap_pairs));
        TRY(enqueue_frame(c, cloud, fc, modes, tc, p, o, zd, scene, views ? &vt : nullptr, t.shutter ? c->sub_frames.p : nullptr));
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

bgs_status bgs_render_ex(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                         const bgs_settings* st, const bgs_render_extras* ex, void* out_rgba, uint32_t out_format,
                         int out_is_device_ptr) {
    return render_impl(c, cloud, view, uni, st, ex, colour_target(&out_rgba, out_format, out_is_device_ptr), nullptr, nullptr, nullptr);
}

bgs_status bgs_render_depth_test(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                                 const bgs_settings* st, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                 void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    return render_impl(c, cloud, view, uni, st, ex, colour_target(&out_rgba, out_format, out_is_device_ptr), depth, nullptr, nullptr);
}

// bgs_render_4d's time refusals (include/bgs.h): time and window finite, time_stop != time_start, and a window length
// that does not overflow
static bgs_status temporal_consts(bgs_context* c, const char* call, float time, float time_start, float time_stop,
                                  TemporalConsts& tc) {
    if (!std::isfinite(time) || !std::isfinite(time_start) || !std::isfinite(time_stop) || time_stop == time_start)
        return fail(c, BGS_EINVAL, "%s: time %g, time_start %g, time_stop %g: all finite and time_stop != time_start", call,
                    (double)time, (double)time_start, (double)time_stop);
    tc.duration = time_stop - time_start;
    if (!std::isfinite(tc.duration)) return fail(c, BGS_EINVAL, "%s: time_stop - time_start overflows", call);
    tc.time = time;
    tc.time_future = time + 1.0e-3f;
    return BGS_OK;
}

bgs_status bgs_render_4d(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                         const bgs_settings* st, const bgs_render_extras* ex, const bgs_scene_depth* depth, void* out_rgba,
                         uint32_t out_format, int out_is_device_ptr, float time_start, float time_stop) {
    if (!c) return BGS_EINVAL;
    TemporalConsts tc = {};
    if (uni) TRY(temporal_consts(c, "render_4d", uni->time, time_start, time_stop, tc));
    return render_impl(c, cloud, view, uni, st, ex, colour_target(&out_rgba, out_format, out_is_device_ptr), depth, &tc, nullptr);
}

// the refusals every scene call makes of its list before reading it: k, SORT_ALL and NULL clouds
// (at most max_k entities: BGS_SCENE_MAX_CLOUDS, or BGS_ENTITIES_MANY_MAX for bgs_render_entities_many)
static bgs_status check_scene_list(bgs_context* c, const char* call, const bgs_cloud* const* clouds, uint32_t k,
                                   const bgs_settings* frame, uint32_t max_k = BGS_SCENE_MAX_CLOUDS) {
    if (k == 0 || k > max_k) return fail(c, BGS_EINVAL, "%s: k = %u is not in 1..%u", call, k, max_k);
    if (frame->flags & BGS_FLAG_SORT_ALL) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_SORT_ALL is not supported", call);
    for (uint32_t j = 0; j < k; ++j)
        if (!clouds[j]) return fail(c, BGS_EINVAL, "%s: clouds[%u] is NULL", call, j);
    return BGS_OK;
}

// the blend kind of an entity's records (raster.cu): 0 = quad-uv, 1 = conic (3DGS and 4D with aabb), 2 = surfel
static int blend_kind(const bgs_entity_settings& e) { return !e.aabb ? 0 : (e.gaussian_mode == BGS_GAUSSIAN_2D ? 2 : 1); }

// a refusal s of entity j's checks, its message led by the entity's index (bgs_render_entities_many: among thousands of
// entities, the message says which)
static bgs_status entity_refusal(bgs_context* c, bgs_status s, const char* call, uint32_t j) {
    char msg[sizeof(c->err)];
    memcpy(msg, c->err, sizeof(msg));
    return fail(c, s, "%s: entities[%u]: %s", call, j, msg);
}

// bgs_render_entities_many's table of k segments in the staging of its slot (bgs_context::many): the slot the last
// frame enqueued with a table did not take, once the frame that last read it has completed; its regions (Layout) as
// SceneTableDev's pointers, in device memory of the context's GPU.  Called once the list has passed every refusal, so a
// refused call neither waits nor allocates.
static bgs_status many_table(bgs_context* c, uint32_t k, SceneFacts* scene) {
    CU(c, cudaSetDevice(c->device));   // (the device copy is the context's GPU's, whatever the thread had current)
    const int slot = c->many_last ^ 1;
    bgs_context::ManySlot& m = c->many[slot];
    if (m.used) CU(c, cudaEventSynchronize(m.ev));
    Layout l;
    const size_t o_seg = l.add((size_t)k * sizeof(SceneSeg)), o_off = l.add((size_t)k * 4);
    const size_t o_times = l.add((size_t)k * sizeof(TemporalConsts)), o_cls = l.add((size_t)k * 4), o_kind = l.add((size_t)k * 4);
    const size_t bytes = l.padded();
    if (bytes > m.host_bytes) {
        if (m.host) cudaFreeHost(m.host);
        m.host = nullptr;
        m.host_bytes = 0;
        CU(c, cudaMallocHost(&m.host, bytes));
        m.host_bytes = bytes;
    }
    TRY(m.dev.grow(c, bytes, false));
    uint8_t* d = m.dev.p;
    scene->many = true;
    scene->slot = slot;
    scene->h_tab = m.host;
    scene->tab_bytes = bytes;
    scene->dtab = SceneTableDev{k, 0u, reinterpret_cast<const SceneSeg*>(d + o_seg), reinterpret_cast<const uint32_t*>(d + o_off),
                                reinterpret_cast<const TemporalConsts*>(d + o_times),
                                reinterpret_cast<const uint32_t*>(d + o_cls), reinterpret_cast<const uint32_t*>(d + o_kind)};
    return BGS_OK;
}

// Every scene frame: k entities, each checked as its single-cloud call (bgs_render_depth_test, or bgs_render_4d for a
// Gaussian4d cloud when with_4d) with its own settings, num_classes and window, drawn into one depth-sorted frame.
// entity_flags: each entity's BGS_ENTITY_* bits (NULL: none).  The list has passed check_scene_list.  Aux targets
// (bgs_render_entities_aux): every segment also projects its Depth and Normal colours, blended into the depth and normal
// frames.  t.v = nv > 1 views (bgs_render_views or, with aux targets, bgs_render_views_aux, which have checked nv, the
// targets and the entities' modes): the k entities seen from each of the nv views (depth: nv buffers, or NULL), segment
// i k + j entity j from view i, view i's frames into its targets.  A shutter frame (t.shutter, bgs_render_shutter, which has
// checked the same): view i is sample i, whose segment i k + j takes uniforms[i k + j] (a views frame's views all take
// uniforms[j]).
static bgs_status render_entities_impl(bgs_context* c, const char* call, bool with_4d, const bgs_cloud* const* clouds,
                                       const bgs_cloud_uniform* unis, const bgs_entity_settings* ents,
                                       const uint32_t* entity_flags, uint32_t k, const bgs_view* view,
                                       const bgs_settings* frame, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                       const Targets& t, bool many = false) {
    const uint32_t nv = t.v;
    // view i's entity j reads unis[i stride + j]; nu sets of uniforms
    const uint32_t stride = t.shutter ? k : 0u, nu = t.shutter ? nv : 1u;
    // each entity's bounding-box overlay: its own bit, or the frame's flag for every entity
    auto box_of = [&](uint32_t j) {
        return (frame->flags & BGS_FLAG_VISUALIZE_BOUNDING_BOX) != 0 ||
               (entity_flags && (entity_flags[j] & BGS_ENTITY_VISUALIZE_BOUNDING_BOX) != 0);
    };
    // entity j as its single-cloud call: its settings with the frame's sort bits and flags, its num_classes and window
    std::vector<bgs_settings> st(k);
    std::vector<TemporalConsts> tcs((size_t)nu * k);   // (entity j's times with uniforms i: tcs[i k + j], Gaussian4d entities only)
    auto scene = std::make_shared<SceneFacts>();
    // (many: a refusal names the entity)
    auto checked = [&](bgs_status s, uint32_t j) { return s == BGS_OK || !many ? s : entity_refusal(c, s, call, j); };
    bool any_depth = false, undrawn = true;
    uint32_t kinds = 0;
    uint64_t total = 0;
    for (uint32_t j = 0; j < k; ++j) {
        const bgs_entity_settings& e = ents[j];
        const bool is4 = with_4d && is_4d(clouds[j]->layout);
        bgs_settings& s = st[j];
        s = *frame;
        s.gaussian_mode = e.gaussian_mode; s.rasterize_mode = e.rasterize_mode; s.aabb = e.aabb;
        s.opacity_adaptive_radius = e.opacity_adaptive_radius; s.draw_mode = e.draw_mode;
        bgs_render_extras ej = ex ? *ex : bgs_render_extras{};
        ej.num_classes = e.num_classes;
        bgs_settings chk = s;   // (a non-4D entity in Velocity is undrawn, and checked as a Color one)
        if (!is4 && chk.rasterize_mode == BGS_RASTERIZE_VELOCITY) chk.rasterize_mode = BGS_RASTERIZE_COLOR;
        for (uint32_t i = 0; i < nv; ++i)   // (as the single-view call of each view)
            TRY(checked(check_render(c, clouds[j], &view[i], &unis[i * stride + j], &chk,
                                     ex || e.rasterize_mode == BGS_RASTERIZE_CLASSIFICATION ? &ej : nullptr, t.format, false, is4,
                                     j == 0 && i == 0),
                        j));
        for (uint32_t i = 0; is4 && i < nu; ++i)
            TRY(checked(temporal_consts(c, call, unis[i * stride + j].time, e.window.time_start, e.window.time_stop, tcs[i * k + j]), j));
        const bgs_entity_settings& e0 = ents[0];
        undrawn = undrawn && !is4 && e.rasterize_mode == BGS_RASTERIZE_VELOCITY && e.gaussian_mode == e0.gaussian_mode &&
                  e.aabb == e0.aabb && e.opacity_adaptive_radius == e0.opacity_adaptive_radius && e.draw_mode == e0.draw_mode &&
                  box_of(j) == box_of(0);
        any_depth = any_depth || e.rasterize_mode == BGS_RASTERIZE_DEPTH;
        kinds |= 1u << blend_kind(e);
        total += clouds[j]->n;
    }
    // (one Velocity frame without a Gaussian4d cloud: nothing has a colour source, as in bgs_render_depth_test)
    if (undrawn) return fail(c, BGS_EINVAL, "%s: a Velocity frame with no Gaussian4d cloud listed", call);
    const uint64_t n_view = total;   // (every view lists the k entities: N = nv x n_view)
    total *= nv;
    if (total >= (1ull << 30)) return fail(c, BGS_EINVAL, "%s: N = %llu gaussians, must be < 2^30", call, (unsigned long long)total);
    if (depth)
        for (uint32_t i = 0; i < nv; ++i) TRY(check_scene_depth(c, &depth[i], &view[i]));
    // where the table goes: the SceneFacts' own arrays, or (many) the staging of a device table
    SceneSeg* segs = scene->tab.seg;
    uint32_t* offsets = scene->kinds.offset;
    TemporalConsts* times = scene->times.t;
    uint32_t* classes = scene->classes.n;
    uint32_t* seg_kinds = scene->kinds.kind;
    if (many) {
        TRY(many_table(c, k, scene.get()));
        uint8_t* h = static_cast<uint8_t*>(const_cast<void*>(scene->h_tab));
        const SceneTableDev& d = scene->dtab;
        const uint8_t* d0 = reinterpret_cast<const uint8_t*>(d.seg);
        segs = reinterpret_cast<SceneSeg*>(h);
        offsets = reinterpret_cast<uint32_t*>(h + (reinterpret_cast<const uint8_t*>(d.offset) - d0));
        times = reinterpret_cast<TemporalConsts*>(h + (reinterpret_cast<const uint8_t*>(d.times) - d0));
        classes = reinterpret_cast<uint32_t*>(h + (reinterpret_cast<const uint8_t*>(d.classes) - d0));
        seg_kinds = reinterpret_cast<uint32_t*>(h + (reinterpret_cast<const uint8_t*>(d.kinds) - d0));
    }
    SceneTable& tab = scene->tab;
    memset(&tab, 0, sizeof(tab));
    tab.k = many ? 1u : k * nv;   // (many: tab holds segment 0 alone, the frame's first)
    tab.n_total = (uint32_t)total;
    scene->kinds.k = many ? 0u : k * nv;
    scene->dtab.n_total = (uint32_t)total;
    uint32_t offset = 0;
    bool box_all = true;
    for (uint32_t i = 0; i < nv; ++i)
        for (uint32_t j = 0; j < k; ++j) {
            const uint32_t sj = i * k + j;   // entity j seen from view i
            const bgs_cloud* cl = clouds[j];
            const uint32_t rm = st[j].rasterize_mode;
            SceneSeg& sg = segs[sj];
            sg.fc = frame_consts(cl, &view[i], &unis[i * stride + j], &st[j], t.aux);
            sg.fc.n_cloud = (uint32_t)n_view;   // (Depth colouring reads its view's sorted list of n_view entries)
            sg.pos = cl->pos;
            sg.blocks = cl->blocks;
            sg.offset = offset;
            sg.n = cl->n;
            // the plain colour kernel, or the Classification / OpticalFlow one (which leaves a 3D Velocity record undrawn)
            sg.group = project_group(cl->layout, cl->sh_degree);
            if (sg.group != PROJECT_GROUP_4D && rm >= BGS_RASTERIZE_CLASSIFICATION) sg.group |= ENTITY_MODES;
            const bool sh = rm == ((sg.group & ENTITY_MODES) ? BGS_RASTERIZE_CLASSIFICATION : BGS_RASTERIZE_COLOR);
            const size_t gi = std::find(scene->groups.begin(), scene->groups.end(), sg.group) - scene->groups.begin();
            if (gi == scene->groups.size()) { scene->groups.push_back(sg.group); scene->need_sh.push_back(0u); }
            if (sh) scene->need_sh[gi] = 1u;
            times[sj] = tcs[(size_t)(stride ? i : 0u) * k + j];
            classes[sj] = ents[j].num_classes;
            offsets[sj] = offset;
            seg_kinds[sj] = (uint32_t)blend_kind(ents[j]) | (box_of(j) ? BOX_KIND : 0u);
            scene->box = scene->box || box_of(j);
            box_all = box_all && box_of(j);
            offset += cl->n;
            scene->clouds.push_back(cl);
        }
    if (many) tab.seg[0] = segs[0];
    scene->distinct = scene->clouds;
    std::sort(scene->distinct.begin(), scene->distinct.end());
    scene->distinct.erase(std::unique(scene->distinct.begin(), scene->distinct.end()), scene->distinct.end());
    if (nv > 1) {   // each view's tiles after the earlier views', its depth buffer
        ViewTable& vt = scene->views;
        vt.v = nv;
        vt.n_view = (uint32_t)n_view;
        for (uint32_t i = 0; i < nv; ++i) {
            const FrameConsts& f = tab.seg[i * k].fc;
            vt.W[i] = f.Wi; vt.H[i] = f.Hi; vt.tiles_x[i] = f.tiles_x; vt.tiles_y[i] = f.tiles_y;
            vt.tile0[i + 1] = vt.tile0[i] + (uint32_t)f.tiles_x * (uint32_t)f.tiles_y;
            if (depth) { vt.scene[i] = depth[i].depth; vt.pitch[i] = (size_t)depth[i].pitch_bytes; }
        }
    }
    // one kind: its own blend; several, or entities with and without the overlay: the mixed one (with the surfel records
    // when some entity has them)
    scene->raster_mode = __builtin_popcount(kinds) > 1 || box_all != scene->box ? ((kinds & 4u) ? 4 : 3) : __builtin_ctz(kinds);
    // the frame as render_impl plans it: its flags and sort bits, the Depth range when some entity is in Depth mode, and
    // the blend kind (an aabb frame when it is not quad-uv: one round)
    bgs_settings sf = *frame;
    sf.rasterize_mode = any_depth ? BGS_RASTERIZE_DEPTH : BGS_RASTERIZE_COLOR;
    sf.aabb = scene->raster_mode != 0;
    sf.gaussian_mode = scene->raster_mode == 2 ? BGS_GAUSSIAN_2D : BGS_GAUSSIAN_3D;
    sf.draw_mode = BGS_DRAW_ALL;
    if (scene->box) sf.flags |= BGS_FLAG_VISUALIZE_BOUNDING_BOX;
    if (nv > 1 || t.pick) sf.flags = (sf.flags & ~(uint32_t)BGS_FLAG_CHUNKS) | BGS_FLAG_NO_CHUNKS;   // (one round)
    return render_impl(c, clouds[0], view, &unis[0], &sf, ex, t, depth, nullptr, scene);
}

// bgs_render_scene, and bgs_render_scene_4d (with_4d: Gaussian4d clouds are projected at uniforms[j].time in windows[j];
// with none listed the two calls are one and windows is not read): the scene's own refusals, then every cloud an entity
// with the frame's settings
static bgs_status render_scene_as_entities(bgs_context* c, const char* call, bool with_4d, const bgs_cloud* const* clouds,
                                           const bgs_cloud_uniform* unis, const bgs_time_window* windows, uint32_t k,
                                           const bgs_view* view, const bgs_settings* st, const bgs_render_extras* ex,
                                           const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format,
                                           int out_is_device_ptr) {
    if (!c) return BGS_EINVAL;
    if (!clouds || !unis || !view || !st) return fail(c, BGS_NOT_READY, "%s: clouds/uniforms/view/settings not ready", call);
    TRY(check_scene_list(c, call, clouds, k, st));
    bool any_4d = false;
    for (uint32_t j = 0; j < k; ++j) any_4d = any_4d || (with_4d && is_4d(clouds[j]->layout));
    if (any_4d) {
        if (!windows) return fail(c, BGS_EINVAL, "%s: windows is NULL with a Gaussian4d cloud listed", call);
        if (st->gaussian_mode == BGS_GAUSSIAN_2D && st->aabb)
            return fail(c, BGS_EINVAL, "%s: BGS_GAUSSIAN_2D with aabb = 1 takes no Gaussian4d cloud (its blend reads a surfel record for every splat)", call);
    }
    // a scene with 4D clouds: those are drawn as bgs_render_4d frames (gaussian_mode read as Gaussian4d), the others with
    // the frame's settings (a Velocity frame's are drawn as nothing, include/bgs.h)
    std::vector<bgs_entity_settings> ents(k);
    for (uint32_t j = 0; j < k; ++j) {
        const bool is4 = any_4d && is_4d(clouds[j]->layout);
        if (any_4d && !is4 && st->gaussian_mode == BGS_GAUSSIAN_4D)
            return fail(c, BGS_EINVAL, "%s: gaussian_mode BGS_GAUSSIAN_4D with clouds[%u], which is not a Gaussian4d cloud", call, j);
        bgs_entity_settings& e = ents[j];
        e.gaussian_mode = is4 ? (uint32_t)BGS_GAUSSIAN_4D : st->gaussian_mode;
        e.rasterize_mode = st->rasterize_mode; e.aabb = st->aabb;
        e.opacity_adaptive_radius = st->opacity_adaptive_radius; e.draw_mode = st->draw_mode;
        e.num_classes = ex ? ex->num_classes : 1u;
        e.window = is4 ? windows[j] : bgs_time_window{};
    }
    return render_entities_impl(c, call, with_4d, clouds, unis, ents.data(), nullptr, k, view, st, ex, depth,
                                colour_target(&out_rgba, out_format, out_is_device_ptr));
}

bgs_status bgs_render_scene(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis, uint32_t k,
                            const bgs_view* view, const bgs_settings* st, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                            void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    return render_scene_as_entities(c, "render_scene", false, clouds, unis, nullptr, k, view, st, ex, depth, out_rgba, out_format,
                                    out_is_device_ptr);
}

bgs_status bgs_render_scene_4d(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                               const bgs_time_window* windows, uint32_t k, const bgs_view* view, const bgs_settings* st,
                               const bgs_render_extras* ex, const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format,
                               int out_is_device_ptr) {
    return render_scene_as_entities(c, "render_scene_4d", true, clouds, unis, windows, k, view, st, ex, depth, out_rgba,
                                    out_format, out_is_device_ptr);
}

// bgs_render_entities_ex's refusals of its arguments before the entities are read as single-cloud calls
static bgs_status check_entities_call(bgs_context* c, const char* call, const bgs_cloud* const* clouds,
                                      const bgs_cloud_uniform* unis, const bgs_entity_settings* ents,
                                      const uint32_t* entity_flags, uint32_t k, const bgs_view* view, const bgs_settings* frame,
                                      uint32_t max_k = BGS_SCENE_MAX_CLOUDS) {
    if (!clouds || !unis || !ents || !view || !frame)
        return fail(c, BGS_NOT_READY, "%s: clouds/uniforms/entities/view/settings not ready", call);
    TRY(check_scene_list(c, call, clouds, k, frame, max_k));
    if (entity_flags)
        for (uint32_t j = 0; j < k; ++j)
            if (entity_flags[j] & ~(uint32_t)BGS_ENTITY_VISUALIZE_BOUNDING_BOX)
                return fail(c, BGS_EINVAL, "%s: entity_flags[%u] = 0x%x has an unknown bit", call, j, entity_flags[j]);
    return BGS_OK;
}

bgs_status bgs_render_entities_ex(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                  const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* view,
                                  const bgs_settings* frame, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                  void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_entities";
    if (!c) return BGS_EINVAL;
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, view, frame));
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth,
                                colour_target(&out_rgba, out_format, out_is_device_ptr));
}

// The refusals of bgs_render_entities_aux, _pick, bgs_render_views and _views_aux (include/bgs.h), in this order, each
// made by the calls it names: bgs_render_entities_ex's of the list; v and v x k (views calls); the targets; BGS_FLAG_ASYNC
// (aux and pick calls); each entity's: Gaussian4d, covariance and Velocity (aux calls), Depth (views without aux),
// OpticalFlow (views calls); blend-over (views calls: device targets only).  A shutter call (bgs_render_shutter, t.shutter)
// makes the views calls' refusals of its v samples, of its one target, and takes blend-over into host targets.
static bgs_status check_targets_call(bgs_context* c, const char* call, const bgs_cloud* const* clouds,
                                     const bgs_cloud_uniform* unis, const bgs_entity_settings* ents,
                                     const uint32_t* entity_flags, uint32_t k, const bgs_view* view, const bgs_settings* frame,
                                     const Targets& t, bool views, bool pick, uint32_t max_k = BGS_SCENE_MAX_CLOUDS) {
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, view, frame, max_k));
    if (views) {
        if (t.v == 0) return fail(c, BGS_EINVAL, "%s: v = 0 views", call);
        if ((uint64_t)t.v * k > BGS_SCENE_MAX_CLOUDS)
            return fail(c, BGS_EINVAL, "%s: v x k = %u x %u segments, at most %d", call, t.v, k, BGS_SCENE_MAX_CLOUDS);
        const size_t bpp = format_bpp(t.format);
        const char* names[3] = {"out_rgba", "out_depth", "out_normal"};
        void* const* arrays[3] = {t.rgba, t.depth, t.normal};
        for (int a = 0; a < (t.aux ? 3 : 1); ++a) {
            if (!arrays[a]) return fail(c, BGS_EINVAL, "%s: %s is NULL", call, names[a]);
            for (uint32_t i = 0; i < (t.shutter ? 1u : t.v); ++i) {
                if (!arrays[a][i]) return fail(c, BGS_EINVAL, "%s: %s[%u] is NULL", call, names[a], i);
                if (t.device && reinterpret_cast<uintptr_t>(arrays[a][i]) % bpp != 0)
                    return fail(c, BGS_EINVAL, "%s: device target %s[%u] = %p is not aligned to its %zu-byte pixels", call,
                                names[a], i, arrays[a][i], bpp);
            }
        }
    } else if (t.aux && (!t.rgba[0] || !t.depth[0] || !t.normal[0])) {
        return fail(c, BGS_EINVAL, "%s: the three output frames are required", call);
    }
    if (pick) {
        if (!t.pick) return fail(c, BGS_EINVAL, "%s: out_pick is NULL", call);
        if (t.device && reinterpret_cast<uintptr_t>(t.pick) % sizeof(bgs_pick) != 0)
            return fail(c, BGS_EINVAL, "%s: device pick target %p is not aligned to its 16-byte records", call, t.pick);
    }
    if ((t.aux || pick) && (frame->flags & BGS_FLAG_ASYNC)) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_ASYNC is not supported", call);
    for (uint32_t j = 0; j < k; ++j) {
        // (a 4D cloud has no Normal colour; a covariance cloud no rotation; Velocity changes which splats draw, and how; a
        // views frame's Depth entity would take its colour range from every view's sorted list; OpticalFlow has one previous
        // view per frame)
        const uint32_t rm = ents[j].rasterize_mode;
        if (t.aux && is_4d(clouds[j]->layout)) return fail(c, BGS_EINVAL, "%s: clouds[%u] is a Gaussian4d cloud", call, j);
        if (t.aux && clouds[j]->layout == CloudLayout::F16Cov)
            return fail(c, BGS_EINVAL, "%s: clouds[%u] is a precomputed-covariance cloud (no rotation for the normal)", call, j);
        if (t.aux && rm == BGS_RASTERIZE_VELOCITY) return fail(c, BGS_EINVAL, "%s: entities[%u] is in Velocity mode", call, j);
        if (views && !t.aux && rm == BGS_RASTERIZE_DEPTH) return fail(c, BGS_EINVAL, "%s: entities[%u] is in Depth mode", call, j);
        if (views && rm == BGS_RASTERIZE_OPTICAL_FLOW)
            return fail(c, BGS_EINVAL, "%s: entities[%u] is in OpticalFlow mode", call, j);
    }
    if (views && !t.shutter && (frame->flags & BGS_FLAG_BLEND_OVER_TARGET) && !t.device)
        return fail(c, BGS_EINVAL, "%s: BGS_FLAG_BLEND_OVER_TARGET takes device targets", call);
    return BGS_OK;
}

// bgs_render_entities_ex's frame and, in the same pass, its Depth and Normal frames (include/bgs.h)
bgs_status bgs_render_entities_aux(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                   const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k,
                                   const bgs_view* view, const bgs_settings* frame, const bgs_render_extras* ex,
                                   const bgs_scene_depth* depth, void* out_rgba, void* out_depth, void* out_normal,
                                   uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_entities_aux";
    if (!c) return BGS_EINVAL;
    const Targets t{out_format, out_is_device_ptr, 1, true, &out_rgba, &out_depth, &out_normal, nullptr};
    TRY(check_targets_call(c, call, clouds, unis, ents, entity_flags, k, view, frame, t, false, false));
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth, t);
}

// bgs_render_entities_ex's frame and, from the same blend, its pick frame (include/bgs.h)
bgs_status bgs_render_entities_pick(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                    const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k,
                                    const bgs_view* view, const bgs_settings* frame, const bgs_render_extras* ex,
                                    const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format, int out_is_device_ptr,
                                    void* out_pick) {
    const char* call = "render_entities_pick";
    if (!c) return BGS_EINVAL;
    const Targets t{out_format, out_is_device_ptr, 1, false, &out_rgba, nullptr, nullptr, out_pick};
    TRY(check_targets_call(c, call, clouds, unis, ents, entity_flags, k, view, frame, t, false, true));
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth, t);
}

// bgs_render_entities_ex and _pick for any number of entities (include/bgs.h): the segment table in device memory
bgs_status bgs_render_entities_many(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                    const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* view,
                                    const bgs_settings* frame, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                    void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_entities_many";
    if (!c) return BGS_EINVAL;
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, view, frame, BGS_ENTITIES_MANY_MAX));
    // (frame_out's refusal, made here so that a refused call has not built the table)
    if (out_is_device_ptr && reinterpret_cast<uintptr_t>(out_rgba) % format_bpp(out_format) != 0)
        return fail(c, BGS_EINVAL, "render: device target %p is not aligned to its %zu-byte pixels", out_rgba, format_bpp(out_format));
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth,
                                colour_target(&out_rgba, out_format, out_is_device_ptr), true);
}

bgs_status bgs_render_entities_pick_many(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                         const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k,
                                         const bgs_view* view, const bgs_settings* frame, const bgs_render_extras* ex,
                                         const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format,
                                         int out_is_device_ptr, void* out_pick) {
    const char* call = "render_entities_pick_many";
    if (!c) return BGS_EINVAL;
    const Targets t{out_format, out_is_device_ptr, 1, false, &out_rgba, nullptr, nullptr, out_pick};
    TRY(check_targets_call(c, call, clouds, unis, ents, entity_flags, k, view, frame, t, false, true, BGS_ENTITIES_MANY_MAX));
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth, t, true);
}

// ---- bgs_entity_list (include/bgs.h): a resident entity list, edited in place, rendered as bgs_render_entities_many

// entity j of an edit as bgs_render_entities_many checks it, in so far as the check depends on the entity alone (the frame's
// format, sort bits, view and OpticalFlow extras are the render call's); x and r its host facts and device record
static bgs_status list_entity(bgs_context* c, const char* call, uint32_t j, const bgs_cloud* cl, const bgs_cloud_uniform& u,
                              const bgs_entity_settings& e, uint32_t flags, ListEntity& x, EntityRec& r, TemporalConsts& tc) {
    if (!cl) return fail(c, BGS_EINVAL, "%s: entities[%u]: the cloud is NULL", call, j);
    if (flags & ~(uint32_t)BGS_ENTITY_VISUALIZE_BOUNDING_BOX)
        return fail(c, BGS_EINVAL, "%s: entities[%u]: entity flags 0x%x have an unknown bit", call, j, flags);
    if (cl->device != c->device) return entity_refusal(c, fail(c, BGS_EINVAL, "render: cloud lives on another device"), call, j);
    const bool is4 = is_4d(cl->layout);
    bgs_settings chk = {};   // (a non-4D entity in Velocity is undrawn, and checked as a Color one)
    chk.gaussian_mode = e.gaussian_mode; chk.aabb = e.aabb; chk.opacity_adaptive_radius = e.opacity_adaptive_radius;
    chk.draw_mode = e.draw_mode;
    chk.rasterize_mode = !is4 && e.rasterize_mode == BGS_RASTERIZE_VELOCITY ? (uint32_t)BGS_RASTERIZE_COLOR : e.rasterize_mode;
    bgs_render_extras ej = {};
    ej.num_classes = e.num_classes;
    const bgs_status s = check_settings(c, cl, &chk, &ej, false, is4, false);
    if (s != BGS_OK) return entity_refusal(c, s, call, j);
    tc = {};
    if (is4) {
        const bgs_status st = temporal_consts(c, call, u.time, e.window.time_start, e.window.time_stop, tc);
        if (st != BGS_OK) return entity_refusal(c, st, call, j);
    }
    uint32_t group = project_group(cl->layout, cl->sh_degree);
    if (group != PROJECT_GROUP_4D && e.rasterize_mode >= BGS_RASTERIZE_CLASSIFICATION) group |= ENTITY_MODES;
    const bool sh = e.rasterize_mode == ((group & ENTITY_MODES) ? BGS_RASTERIZE_CLASSIFICATION : BGS_RASTERIZE_COLOR);
    x = ListEntity{cl, u, e, flags, cl->n, group, 0u, sh, is4};
    r = EntityRec{u, e.gaussian_mode, e.rasterize_mode, e.aabb, e.opacity_adaptive_radius, e.draw_mode, cl->n, group,
                  cl->layout == CloudLayout::F16Cov ? 1u : 0u, cl->pos, cl->blocks};
    return BGS_OK;
}

// the key render_entities_impl's Velocity refusal compares entities by (box: the entity's overlay bit as the frame sees it)
static std::array<uint32_t, 5> velocity_key(const ListEntity& x, bool box) {
    return {x.e.gaussian_mode, x.e.aabb, x.e.opacity_adaptive_radius, x.e.draw_mode, box ? 1u : 0u};
}

// adds (d = +1) or removes (d = -1) entity x's share of the list's counters
static void list_count(bgs_entity_list* l, const ListEntity& x, int d) {
    auto bump = [d](uint32_t& v) { v = (uint32_t)((int64_t)v + d); };
    if (x.cloud) {
        if ((l->clouds[x.cloud] += (uint32_t)d) == 0) l->clouds.erase(x.cloud);
    } else {
        bump(l->detached);
    }
    std::array<uint32_t, 2>& g = l->groups[x.group];
    bump(g[0]);
    if (x.sh) bump(g[1]);
    if (g[0] == 0) l->groups.erase(x.group);
    bump(l->kinds[blend_kind(x.e)]);
    const bool boxed = (x.flags & BGS_ENTITY_VISUALIZE_BOUNDING_BOX) != 0;
    if (boxed) bump(l->boxed);
    if (x.e.rasterize_mode == BGS_RASTERIZE_DEPTH) bump(l->depth);
    if (x.e.rasterize_mode == BGS_RASTERIZE_OPTICAL_FLOW) bump(l->flow);
    if (!x.is4 && x.e.rasterize_mode == BGS_RASTERIZE_VELOCITY)
        for (int b = 0; b < 2; ++b) {
            const auto key = velocity_key(x, b ? true : boxed);
            if ((l->velocity[b][key] += (uint32_t)d) == 0) l->velocity[b].erase(key);
        }
    l->total = (uint64_t)((int64_t)l->total + d * (int64_t)x.n);
}

// the list's current generation, writable for entities [0, need): written in place when no frame holds it; else (or when
// it is too small) the list moves to a generation no frame holds, a held one kept as the spare, with [0, size) copied
// over on the context's stream (after every frame that read the generation it moves to)
static bgs_status list_writable(bgs_entity_list* l, uint32_t need) {
    bgs_context* c = l->ctx;
    std::shared_ptr<ListTable>& cur = l->cur;
    if (cur && cur.use_count() == 1 && cur->cap >= need) return BGS_OK;
    std::shared_ptr<ListTable> next;
    if (l->spare && l->spare.use_count() == 1 && l->spare->cap >= need) {
        next = l->spare;
    } else {
        const uint32_t cap = std::max({need, 64u, cur ? std::min(2u * cur->cap, BGS_ENTITIES_MANY_MAX) : 0u});
        next = std::make_shared<ListTable>();
        Layout lay;
        const size_t o_rec = lay.add((size_t)cap * sizeof(EntityRec)), o_off = lay.add((size_t)cap * 4);
        const size_t o_t = lay.add((size_t)cap * sizeof(TemporalConsts)), o_cls = lay.add((size_t)cap * 4);
        const size_t o_k = lay.add((size_t)cap * 4), o_kb = lay.add((size_t)cap * 4), o_seg = lay.add((size_t)cap * sizeof(SceneSeg));
        TRY(next->mem.grow(c, lay.padded(), false));
        uint8_t* m = next->mem.p;
        next->cap = cap;
        next->a = EntityListArrays{reinterpret_cast<EntityRec*>(m + o_rec), reinterpret_cast<uint32_t*>(m + o_off),
                                   reinterpret_cast<TemporalConsts*>(m + o_t), reinterpret_cast<uint32_t*>(m + o_cls),
                                   reinterpret_cast<uint32_t*>(m + o_k), reinterpret_cast<uint32_t*>(m + o_kb)};
        next->seg = reinterpret_cast<SceneSeg*>(m + o_seg);
    }
    const size_t k = l->ent.size();
    if (cur && k) {
        const EntityListArrays &f = cur->a, &t = next->a;
        cudaStream_t q = c->stream;
        CU(c, cudaMemcpyAsync(t.recs, f.recs, k * sizeof(EntityRec), cudaMemcpyDeviceToDevice, q));
        CU(c, cudaMemcpyAsync(t.offset, f.offset, k * 4, cudaMemcpyDeviceToDevice, q));
        CU(c, cudaMemcpyAsync(t.times, f.times, k * sizeof(TemporalConsts), cudaMemcpyDeviceToDevice, q));
        CU(c, cudaMemcpyAsync(t.classes, f.classes, k * 4, cudaMemcpyDeviceToDevice, q));
        CU(c, cudaMemcpyAsync(t.kinds, f.kinds, k * 4, cudaMemcpyDeviceToDevice, q));
        CU(c, cudaMemcpyAsync(t.kinds_box, f.kinds_box, k * 4, cudaMemcpyDeviceToDevice, q));
    }
    l->spare = cur && cur.use_count() > 1 ? cur : (next == l->spare ? nullptr : l->spare);
    cur = next;
    return BGS_OK;
}

// the edit of entities idx[0 .. count) (each < the size, distinct; idx == NULL: an append after the last entity) to the
// given ones: every entity checked before anything changes, then the counters, the host facts and, in one upload and one
// scatter, the device arrays; the offsets after the first entity whose gaussian count changed are rewritten (O(k))
static bgs_status list_edit(bgs_entity_list* l, const char* call, const uint32_t* idx, uint32_t count,
                            const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis, const bgs_entity_settings* ents,
                            const uint32_t* entity_flags) {
    if (!l || !l->ctx) return BGS_EINVAL;
    bgs_context* c = l->ctx;
    const uint32_t k = (uint32_t)l->ent.size();
    if (!idx && (uint64_t)k + count > BGS_ENTITIES_MANY_MAX)
        return fail(c, BGS_EINVAL, "%s: k = %llu entities, at most %u", call, (unsigned long long)k + count, BGS_ENTITIES_MANY_MAX);
    if (count == 0) return BGS_OK;
    if (!clouds || !unis || !ents) return fail(c, BGS_EINVAL, "%s: clouds/uniforms/entities is NULL", call);
    CU(c, cudaSetDevice(c->device));
    if (idx) {
        std::vector<uint32_t> sorted(idx, idx + count);
        std::sort(sorted.begin(), sorted.end());
        if (sorted.back() >= k) return fail(c, BGS_EINVAL, "%s: index %u is not below k = %u", call, sorted.back(), k);
        if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
            return fail(c, BGS_EINVAL, "%s: index %u is given twice", call, *std::adjacent_find(sorted.begin(), sorted.end()));
    }
    // the upload: idx | records | offsets | times | num_classes | kinds
    Layout lay;
    const size_t o_idx = lay.add((size_t)count * 4), o_rec = lay.add((size_t)count * sizeof(EntityRec));
    const size_t o_off = lay.add((size_t)count * 4), o_t = lay.add((size_t)count * sizeof(TemporalConsts));
    const size_t o_cls = lay.add((size_t)count * 4), o_k = lay.add((size_t)count * 4);
    std::vector<uint8_t> up(lay.padded());
    uint32_t* u_idx = reinterpret_cast<uint32_t*>(up.data() + o_idx);
    EntityRec* u_rec = reinterpret_cast<EntityRec*>(up.data() + o_rec);
    uint32_t* u_off = reinterpret_cast<uint32_t*>(up.data() + o_off);
    TemporalConsts* u_t = reinterpret_cast<TemporalConsts*>(up.data() + o_t);
    uint32_t* u_cls = reinterpret_cast<uint32_t*>(up.data() + o_cls);
    uint32_t* u_k = reinterpret_cast<uint32_t*>(up.data() + o_k);
    std::vector<ListEntity> xs(count);
    int64_t total = (int64_t)l->total;
    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t j = idx ? idx[i] : k + i;
        const uint32_t f = entity_flags ? entity_flags[i] : 0u;
        TRY(list_entity(c, call, j, clouds[i], unis[i], ents[i], f, xs[i], u_rec[i], u_t[i]));
        u_idx[i] = j;
        u_cls[i] = ents[i].num_classes;
        u_k[i] = (uint32_t)blend_kind(ents[i]) | ((f & BGS_ENTITY_VISUALIZE_BOUNDING_BOX) ? BOX_KIND : 0u);
        total += (int64_t)xs[i].n - (idx ? (int64_t)l->ent[j].n : 0);
    }
    if (total >= (1ll << 30)) return fail(c, BGS_EINVAL, "%s: N = %lld gaussians, must be < 2^30", call, (long long)total);
    TRY(list_writable(l, k + (idx ? 0u : count)));
    TRY(l->upload.grow(c, up.size(), false));
    std::lock_guard<std::mutex> lk(g_registry_mu);   // (bgs_cloud_destroy detaches entities under it)
    uint32_t moved = k;   // the first entity whose gaussian count changed
    if (!idx) l->ent.resize(k + count);
    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t j = u_idx[i];
        if (idx) {
            if (l->ent[j].n != xs[i].n) moved = std::min(moved, j);
            list_count(l, l->ent[j], -1);
        }
        xs[i].offset = idx ? l->ent[j].offset : (uint32_t)(j ? l->ent[j - 1].offset + l->ent[j - 1].n : 0u);
        l->ent[j] = xs[i];
        list_count(l, xs[i], +1);
    }
    std::vector<uint32_t> offsets;
    if (moved < k) {
        for (uint32_t j = moved; j < (uint32_t)l->ent.size(); ++j) {
            l->ent[j].offset = j ? l->ent[j - 1].offset + l->ent[j - 1].n : 0u;
            offsets.push_back(l->ent[j].offset);
        }
    }
    for (uint32_t i = 0; i < count; ++i) u_off[i] = l->ent[u_idx[i]].offset;
    cudaStream_t q = c->stream;
    // (pageable sources: each copy has taken its bytes when it returns, so the vectors may go)
    CU(c, cudaMemcpyAsync(l->upload.p, up.data(), up.size(), cudaMemcpyHostToDevice, q));
    const uint8_t* d = l->upload.p;
    const EntityListUpload u{reinterpret_cast<const uint32_t*>(d + o_idx), reinterpret_cast<const EntityRec*>(d + o_rec),
                             reinterpret_cast<const uint32_t*>(d + o_off), reinterpret_cast<const TemporalConsts*>(d + o_t),
                             reinterpret_cast<const uint32_t*>(d + o_cls), reinterpret_cast<const uint32_t*>(d + o_k)};
    CU(c, launch_entity_list_scatter(u, count, l->cur->a, q));
    if (!offsets.empty())
        CU(c, cudaMemcpyAsync(l->cur->a.offset + moved, offsets.data(), offsets.size() * 4, cudaMemcpyHostToDevice, q));
    return BGS_OK;
}

bgs_status bgs_entity_list_create(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                  const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k,
                                  bgs_entity_list** out) {
    if (!c || !out) return BGS_EINVAL;
    *out = nullptr;
    bgs_entity_list* l = new (std::nothrow) bgs_entity_list();
    if (!l) return fail(c, BGS_ENOMEM, "entity_list_create: out of host memory");
    l->ctx = c;
    const bgs_status s = list_edit(l, "entity_list_create", nullptr, k, clouds, unis, ents, entity_flags);
    if (s != BGS_OK) {
        delete l;
        return s;
    }
    std::lock_guard<std::mutex> lk(g_registry_mu);
    g_lists.push_back(l);
    *out = l;
    return BGS_OK;
}

bgs_status bgs_entity_list_set(bgs_entity_list* l, const uint32_t* indices, uint32_t count, const bgs_cloud* const* clouds,
                               const bgs_cloud_uniform* unis, const bgs_entity_settings* ents, const uint32_t* entity_flags) {
    if (!l || !l->ctx) return BGS_EINVAL;
    if (count && !indices) return fail(l->ctx, BGS_EINVAL, "entity_list_set: indices is NULL");
    return list_edit(l, "entity_list_set", count ? indices : nullptr, count, clouds, unis, ents, entity_flags);
}

bgs_status bgs_entity_list_append(bgs_entity_list* l, uint32_t count, const bgs_cloud* const* clouds,
                                  const bgs_cloud_uniform* unis, const bgs_entity_settings* ents, const uint32_t* entity_flags) {
    return list_edit(l, "entity_list_append", nullptr, count, clouds, unis, ents, entity_flags);
}

bgs_status bgs_entity_list_truncate(bgs_entity_list* l, uint32_t k) {
    if (!l || !l->ctx) return BGS_EINVAL;
    if (k > l->ent.size()) return fail(l->ctx, BGS_EINVAL, "entity_list_truncate: k = %u is above the size %zu", k, l->ent.size());
    std::lock_guard<std::mutex> lk(g_registry_mu);
    for (size_t j = k; j < l->ent.size(); ++j) list_count(l, l->ent[j], -1);
    l->ent.resize(k);   // (the device arrays past k are not read)
    return BGS_OK;
}

bgs_status bgs_entity_list_set_transforms(bgs_entity_list* l, uint32_t first, uint32_t count, const float* m, uint32_t layout,
                                          int is_device_ptr) {
    const char* call = "entity_list_set_transforms";
    if (!l || !l->ctx) return BGS_EINVAL;
    bgs_context* c = l->ctx;
    if ((uint64_t)first + count > l->ent.size())
        return fail(c, BGS_EINVAL, "%s: [%u, %llu) is beyond the size %zu", call, first, (unsigned long long)first + count, l->ent.size());
    if (layout != BGS_MATRIX_COLUMN_MAJOR && layout != BGS_MATRIX_ROW_MAJOR) return fail(c, BGS_EINVAL, "%s: unknown layout %u", call, layout);
    if (count == 0) return BGS_OK;
    if (!m) return fail(c, BGS_EINVAL, "%s: m is NULL", call);
    CU(c, cudaSetDevice(c->device));
    if (is_device_ptr) {
        cudaPointerAttributes a = {};
        const cudaError_t e = cudaPointerGetAttributes(&a, m);
        if (e != cudaSuccess) cudaGetLastError();   // (an unknown pointer: clear the error, refuse below)
        if (e != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != c->device)
            return fail(c, BGS_EINVAL, "%s: m = %p is not device memory of device %d", call, (const void*)m, c->device);
    }
    TRY(list_writable(l, (uint32_t)l->ent.size()));
    cudaStream_t q = c->stream;
    const size_t bytes = (size_t)count * 64;
    const float* src = m;
    if (!is_device_ptr) {
        // host matrices go through the upload buffer from a copy of the library's own, so the caller's array (pageable or
        // pinned) may be reused once the call returns
        TRY(l->upload.grow(c, bytes, false));
        const std::vector<float> staged(m, m + (size_t)count * 16);
        CU(c, cudaMemcpyAsync(l->upload.p, staged.data(), bytes, cudaMemcpyHostToDevice, q));   // (pageable: taken on return)
        src = reinterpret_cast<const float*>(l->upload.p);
    }
    EntityRec* dst = l->cur->a.recs + first;
    if (layout == BGS_MATRIX_ROW_MAJOR) CU(c, launch_entity_list_transforms(src, count, dst, q));
    else CU(c, cudaMemcpy2DAsync(dst->uni.transform, sizeof(EntityRec), src, 64, 64, count, cudaMemcpyDeviceToDevice, q));
    if (!is_device_ptr)   // (once nothing can fail)
        for (uint32_t i = 0; i < count; ++i)
            for (int e = 0; e < 16; ++e)
                l->ent[first + i].uni.transform[e] = layout == BGS_MATRIX_ROW_MAJOR ? m[i * 16 + (e & 3) * 4 + (e >> 2)] : m[i * 16 + e];
    return BGS_OK;
}

uint32_t bgs_entity_list_size(const bgs_entity_list* l) { return l ? (uint32_t)l->ent.size() : 0u; }

void bgs_entity_list_destroy(bgs_entity_list* l) {
    if (!l) return;
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);
        g_lists.erase(std::remove(g_lists.begin(), g_lists.end(), l), g_lists.end());
        if (bgs_context* c = l->ctx) {
            cudaSetDevice(c->device);
            if (c->async_pending) c->each_stream([](cudaStream_t& s, int) { cudaStreamSynchronize(s); });
            for (FrameFacts* f : {&c->pend, &c->last})
                if (f->scene && f->scene->list == l) {
                    if (f == &c->last) c->have_frame = false;
                    f->forget();
                    f->n = 0;
                }
        }
    }
    delete l;   // (its generations go once no frame holds them)
}

// bgs_render_entity_list and _pick: the refusals bgs_render_entities_many / _pick_many would make of the list that depend
// on the frame, then the frame's facts from the list's counters and its expansion over the list's current generation
static bgs_status render_list_impl(bgs_context* c, const char* call, const bgs_entity_list* l, const bgs_view* view,
                                   const bgs_settings* frame, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                   const Targets& t) {
    if (!c || !l) return BGS_EINVAL;
    if (l->ctx != c) return fail(c, BGS_EINVAL, "%s: the list belongs to another context", call);
    if (!view || !frame) return fail(c, BGS_NOT_READY, "%s: view/settings not ready", call);
    const uint32_t k = (uint32_t)l->ent.size();
    if (k == 0) return fail(c, BGS_EINVAL, "%s: k = 0 is not in 1..%u", call, BGS_ENTITIES_MANY_MAX);
    if (frame->flags & BGS_FLAG_SORT_ALL) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_SORT_ALL is not supported", call);
    CU(c, cudaSetDevice(c->device));
    auto scene = std::make_shared<SceneFacts>();
    const bool box_frame = (frame->flags & BGS_FLAG_VISUALIZE_BOUNDING_BOX) != 0;
    bool undrawn;
    {
        std::lock_guard<std::mutex> lk(g_registry_mu);   // (the counters, against a detaching bgs_cloud_destroy)
        if (l->detached) {
            uint32_t j = 0;
            while (l->ent[j].cloud) ++j;
            return fail(c, BGS_EINVAL, "%s: entities[%u]: its cloud was destroyed (bgs_entity_list_set replaces it)", call, j);
        }
        const ListEntity& x0 = l->ent[0];
        undrawn = !x0.is4 && x0.e.rasterize_mode == BGS_RASTERIZE_VELOCITY;
        if (undrawn) {
            const auto& counts = l->velocity[box_frame ? 1 : 0];
            const auto it = counts.find(velocity_key(x0, box_frame || (x0.flags & BGS_ENTITY_VISUALIZE_BOUNDING_BOX)));
            undrawn = it != counts.end() && it->second == k;
        }
        for (const auto& cl : l->clouds) scene->distinct.push_back(cl.first);
        for (const auto& g : l->groups) {
            scene->groups.push_back(g.first);
            scene->need_sh.push_back(g.second[1] ? 1u : 0u);
        }
        scene->box = box_frame || l->boxed > 0;
        const bool box_all = box_frame || l->boxed == k;
        const uint32_t kinds = (l->kinds[0] ? 1u : 0u) | (l->kinds[1] ? 2u : 0u) | (l->kinds[2] ? 4u : 0u);
        scene->raster_mode = __builtin_popcount(kinds) > 1 || box_all != scene->box ? ((kinds & 4u) ? 4 : 3) : __builtin_ctz(kinds);
        // segment 0 as the host keeps it: render_impl and enqueue_frame read only its frame-wide fields (view, tiles, sort
        // bits, aux) and its rasterize_mode, never the transform, which may have been set from device memory since
        SceneSeg& s0 = scene->tab.seg[0];
        bgs_settings st0 = *frame;
        st0.gaussian_mode = x0.e.gaussian_mode; st0.rasterize_mode = x0.e.rasterize_mode; st0.aabb = x0.e.aabb;
        st0.opacity_adaptive_radius = x0.e.opacity_adaptive_radius; st0.draw_mode = x0.e.draw_mode;
        TRY(check_frame_bits(c, frame, t.format));
        TRY(check_viewport(c, view));
        s0.fc = frame_consts(x0.cloud, view, &x0.uni, &st0, false);
        s0.fc.n_cloud = (uint32_t)l->total;
        s0.pos = x0.cloud->pos; s0.blocks = x0.cloud->blocks; s0.offset = 0; s0.n = x0.n; s0.group = x0.group;
        scene->tab.k = 1;
        scene->tab.n_total = (uint32_t)l->total;
        scene->many = true;
        scene->list = l;
        scene->list_tab = l->cur;
        scene->list_view = *view;
        scene->list_depth_bits = frame->radix_sort_depth_bits;
        const ListTable& lt = *l->cur;
        scene->dtab = SceneTableDev{k, (uint32_t)l->total, lt.seg, lt.a.offset, lt.a.times, lt.a.classes,
                                    box_frame ? lt.a.kinds_box : lt.a.kinds};
        if (l->flow) TRY(check_flow_extras(c, ex));
    }
    if (undrawn) return fail(c, BGS_EINVAL, "%s: a Velocity frame with no Gaussian4d cloud listed", call);
    if (depth) TRY(check_scene_depth(c, depth, view));
    if (t.device && reinterpret_cast<uintptr_t>(t.rgba[0]) % format_bpp(t.format) != 0)
        return fail(c, BGS_EINVAL, "render: device target %p is not aligned to its %zu-byte pixels", t.rgba[0], format_bpp(t.format));
    if (t.pick) {
        if (t.device && reinterpret_cast<uintptr_t>(t.pick) % sizeof(bgs_pick) != 0)
            return fail(c, BGS_EINVAL, "%s: device pick target %p is not aligned to its 16-byte records", call, t.pick);
        if (frame->flags & BGS_FLAG_ASYNC) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_ASYNC is not supported", call);
    }
    // the frame as render_entities_impl plans it
    bgs_settings sf = *frame;
    sf.rasterize_mode = l->depth ? BGS_RASTERIZE_DEPTH : BGS_RASTERIZE_COLOR;
    sf.aabb = scene->raster_mode != 0;
    sf.gaussian_mode = scene->raster_mode == 2 ? BGS_GAUSSIAN_2D : BGS_GAUSSIAN_3D;
    sf.draw_mode = BGS_DRAW_ALL;
    if (scene->box) sf.flags |= BGS_FLAG_VISUALIZE_BOUNDING_BOX;
    if (t.pick) sf.flags = (sf.flags & ~(uint32_t)BGS_FLAG_CHUNKS) | BGS_FLAG_NO_CHUNKS;   // (one round)
    return render_impl(c, l->ent[0].cloud, view, &l->ent[0].uni, &sf, ex, t, depth, nullptr, scene);
}

bgs_status bgs_render_entity_list(bgs_context* c, const bgs_entity_list* l, const bgs_view* view, const bgs_settings* frame,
                                  const bgs_render_extras* ex, const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format,
                                  int out_is_device_ptr) {
    return render_list_impl(c, "render_entity_list", l, view, frame, ex, depth, colour_target(&out_rgba, out_format, out_is_device_ptr));
}

bgs_status bgs_render_entity_list_pick(bgs_context* c, const bgs_entity_list* l, const bgs_view* view, const bgs_settings* frame,
                                       const bgs_render_extras* ex, const bgs_scene_depth* depth, void* out_rgba,
                                       uint32_t out_format, int out_is_device_ptr, void* out_pick) {
    const char* call = "render_entity_list_pick";
    if (c && !out_pick) return fail(c, BGS_EINVAL, "%s: out_pick is NULL", call);
    const Targets t{out_format, out_is_device_ptr, 1, false, &out_rgba, nullptr, nullptr, out_pick};
    return render_list_impl(c, call, l, view, frame, ex, depth, t);
}

// bgs_render_entities_ex of each of v views in one frame (include/bgs.h); one view is bgs_render_entities_ex itself
bgs_status bgs_render_views(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                            const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* views,
                            uint32_t v, const bgs_settings* frame, const bgs_scene_depth* depths, void* const* out_rgba,
                            uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_views";
    if (!c) return BGS_EINVAL;
    const Targets t{out_format, out_is_device_ptr, v, false, out_rgba, nullptr, nullptr, nullptr};
    TRY(check_targets_call(c, call, clouds, unis, ents, entity_flags, k, views, frame, t, true, false));
    if (v == 1)
        return bgs_render_entities_ex(c, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, out_rgba[0], out_format,
                                      out_is_device_ptr);
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, t);
}

// bgs_render_entities_aux of each of v views in one frame (include/bgs.h); one view is bgs_render_entities_aux itself
bgs_status bgs_render_views_aux(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* views,
                                uint32_t v, const bgs_settings* frame, const bgs_scene_depth* depths, void* const* out_rgba,
                                void* const* out_depth, void* const* out_normal, uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_views_aux";
    if (!c) return BGS_EINVAL;
    const Targets t{out_format, out_is_device_ptr, v, true, out_rgba, out_depth, out_normal, nullptr};
    TRY(check_targets_call(c, call, clouds, unis, ents, entity_flags, k, views, frame, t, true, false));
    if (v == 1)
        return bgs_render_entities_aux(c, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, out_rgba[0],
                                       out_depth[0], out_normal[0], out_format, out_is_device_ptr);
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, t);
}

// The mean of s sub-frames of bgs_render_entities_ex, each with its own view and uniforms, in one frame (include/bgs.h);
// one sample is bgs_render_entities_ex itself
bgs_status bgs_render_shutter(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                              const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* views,
                              uint32_t s, const bgs_settings* frame, const bgs_scene_depth* depths, void* out_rgba,
                              uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_shutter";
    if (!c) return BGS_EINVAL;
    Targets t = colour_target(&out_rgba, out_format, out_is_device_ptr);
    t.v = s;
    t.shutter = true;
    TRY(check_targets_call(c, call, clouds, unis, ents, entity_flags, k, views, frame, t, true, false));
    for (uint32_t i = 1; i < s; ++i)
        if ((int)views[i].viewport[2] != (int)views[0].viewport[2] || (int)views[i].viewport[3] != (int)views[0].viewport[3])
            return fail(c, BGS_EINVAL, "%s: views[%u] is %dx%d, views[0] %dx%d: every sample is one frame's size", call, i,
                        (int)views[i].viewport[2], (int)views[i].viewport[3], (int)views[0].viewport[2], (int)views[0].viewport[3]);
    if (s == 1)
        return bgs_render_entities_ex(c, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, out_rgba, out_format,
                                      out_is_device_ptr);
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, t);
}

bgs_status bgs_render_entities(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                               const bgs_entity_settings* ents, uint32_t k, const bgs_view* view, const bgs_settings* frame,
                               const bgs_render_extras* ex, const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format,
                               int out_is_device_ptr) {
    return bgs_render_entities_ex(c, clouds, unis, ents, nullptr, k, view, frame, ex, depth, out_rgba, out_format,
                                  out_is_device_ptr);
}

bgs_status bgs_render(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                      const bgs_settings* st, void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    return bgs_render_ex(c, cloud, view, uni, st, nullptr, out_rgba, out_format, out_is_device_ptr);
}

bgs_status bgs_render_aux(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                          const bgs_settings* st, void* out_rgba, void* out_depth, void* out_normal, uint32_t out_format,
                          int out_is_device_ptr) {
    if (c && (!out_rgba || !out_depth || !out_normal)) return fail(c, BGS_EINVAL, "render_aux: the three output frames are required");
    if (c && st && (st->flags & BGS_FLAG_ASYNC)) return fail(c, BGS_EINVAL, "render_aux: BGS_FLAG_ASYNC is not supported");
    const Targets t{out_format, out_is_device_ptr, 1, true, &out_rgba, &out_depth, &out_normal, nullptr};
    return render_impl(c, cloud, view, uni, st, nullptr, t, nullptr, nullptr, nullptr);
}

bgs_status bgs_debug_sorted_entries(bgs_context* c, uint32_t* out) {
    if (!c || !out) return BGS_EINVAL;
    if (!c->have_frame || !c->last.cloud) return fail(c, BGS_NOT_READY, "no frame rendered yet");
    CU(c, cudaSetDevice(c->device));
    const uint32_t n = c->last.n, n_vis = c->stats.n_visible;
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
        if (c->last.scene && c->last.scene->many) launch_culled_flags_many(c->last.scene->dtab, flags, c->stream);
        else if (c->last.scene) launch_culled_flags_scene(c->last.scene->tab, flags, c->stream);
        else launch_culled_flags(c->last.cloud->pos, n, c->last.fc, flags, c->stream);
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

bgs_status bgs_debug_splat_depths(bgs_context* c, float* out) {
    if (!c || !out) return BGS_EINVAL;
    if (!c->have_frame || !c->last.depth_tested) return fail(c, BGS_NOT_READY, "no depth-tested frame rendered yet");
    CU(c, cudaSetDevice(c->device));
    const uint32_t n_vis = c->stats.n_visible;
    std::vector<float> d(n_vis);
    CU(c, cudaMemcpy(d.data(), c->splat_depth.p, (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
    if (!c->last.by_slot) { std::copy(d.begin(), d.end(), out); return BGS_OK; }
    std::vector<uint32_t> v(n_vis);   // compact frames: rank r's record is at the slot the sort put at n_vis - 1 - r
    CU(c, cudaMemcpy(v.data(), c->vals[c->depth_result].p, (size_t)n_vis * 4, cudaMemcpyDeviceToHost));
    for (uint32_t r = 0; r < n_vis; ++r) out[r] = d[v[n_vis - 1 - r]];
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
