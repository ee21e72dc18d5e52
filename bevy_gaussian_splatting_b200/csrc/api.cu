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
    // a views frame: view i's device targets, host frames (host targets; else NULL) and bytes (of one frame); the depth and
    // normal ones on aux frames
    uint32_t views = 0;
    void* view_rgba[MAX_VIEWS] = {};
    void* view_host[MAX_VIEWS] = {};
    void* view_depth[MAX_VIEWS] = {};
    void* view_normal[MAX_VIEWS] = {};
    void* view_host_depth[MAX_VIEWS] = {};
    void* view_host_normal[MAX_VIEWS] = {};
    size_t view_bytes[MAX_VIEWS] = {};
    // a pick frame (bgs_render_entities_pick): its device records, the host target they are copied to (else NULL)
    uint4* pick = nullptr;
    void* host_pick = nullptr;
};

// A views frame's targets: view i's frame into rgba[i] and, on aux frames, its depth and normal frames into depth[i] and
// normal[i] (NULL arrays otherwise)
struct ViewTargets {
    void* const* rgba;
    void* const* depth;
    void* const* normal;
};

// the caller's device frames, or the library's own (grown on demand)
bgs_status frame_out(bgs_context* c, const bgs_settings* st, uint32_t format, size_t bytes, void* out_rgba,
                     int out_is_device_ptr, bool want_aux, void* out_depth, void* out_normal, FrameOut* o) {
    const bool blend_over = (st->flags & BGS_FLAG_BLEND_OVER_TARGET) != 0;
    o->raster_format = format | ((blend_over ? 2u : ((st->flags & BGS_FLAG_PREMULTIPLIED_OUT) ? 1u : 0u)) << 8);
    o->bytes = bytes;
    // device targets are written with pixel-sized vector stores (and read so in blend-over mode): each must be aligned to
    // one pixel, 4 / 8 / 16 bytes
    const size_t bpp = format_bpp(format);
    if (out_is_device_ptr)
        for (const void* t : {out_rgba, want_aux ? out_depth : nullptr, want_aux ? out_normal : nullptr})
            if (reinterpret_cast<uintptr_t>(t) % bpp != 0)
                return fail(c, BGS_EINVAL, "render: device target %p is not aligned to its %zu-byte pixels", t, bpp);
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
        // (blend-over, queued or not, keeps blending into the frame the previous call produced; synchronous calls that do
        // not blend over use frame 0)
        int k = 0;
        if (blend_over) k = c->frame_last;
        else if (st->flags & BGS_FLAG_ASYNC) { k = c->frame_toggle; c->frame_toggle ^= 1; }
        c->frame_last = k;
        if (st->flags & BGS_FLAG_ASYNC) o->slot = k;
        o->rgba = c->frames[k].p;
        o->host_rgba = out_rgba;
    }
    if (!want_aux) return BGS_OK;
    if (out_is_device_ptr) { o->depth = out_depth; o->normal = out_normal; return BGS_OK; }
    for (int k = 0; k < 2; ++k) TRY(c->frame_aux[k].grow(c, bytes, true));
    o->depth = c->frame_aux[0].p; o->normal = c->frame_aux[1].p;
    o->host_depth = out_depth; o->host_normal = out_normal;
    return BGS_OK;
}

// a views frame's targets: the caller's device frames, or the library's frames holding every view, one after another
// (aux frames: frame_aux[0] every view's depth frame, frame_aux[1] every normal frame) (the targets have passed
// bgs_render_views' or bgs_render_views_aux's checks)
bgs_status frame_out_views(bgs_context* c, const bgs_settings* st, uint32_t format, const ViewTable& vt, const ViewTargets& t,
                           int out_is_device_ptr, FrameOut* o) {
    const size_t bpp = format_bpp(format);
    const bool aux = t.depth != nullptr;
    size_t total = 0;
    for (uint32_t i = 0; i < vt.v; ++i) total += (size_t)vt.W[i] * vt.H[i] * bpp;
    TRY(frame_out(c, st, format, out_is_device_ptr ? (size_t)vt.W[0] * vt.H[0] * bpp : total,
                  out_is_device_ptr ? t.rgba[0] : nullptr, out_is_device_ptr, false, nullptr, nullptr, o));
    if (aux && !out_is_device_ptr)
        for (int k = 0; k < 2; ++k) TRY(c->frame_aux[k].grow(c, total, true));
    o->views = vt.v;
    size_t at = 0;
    for (uint32_t i = 0; i < vt.v; ++i) {
        o->view_bytes[i] = (size_t)vt.W[i] * vt.H[i] * bpp;
        o->view_rgba[i] = out_is_device_ptr ? t.rgba[i] : static_cast<char*>(o->rgba) + at;
        o->view_host[i] = out_is_device_ptr ? nullptr : t.rgba[i];
        if (aux) {
            o->view_depth[i] = out_is_device_ptr ? t.depth[i] : static_cast<char*>(c->frame_aux[0].p) + at;
            o->view_normal[i] = out_is_device_ptr ? t.normal[i] : static_cast<char*>(c->frame_aux[1].p) + at;
            o->view_host_depth[i] = out_is_device_ptr ? nullptr : t.depth[i];
            o->view_host_normal[i] = out_is_device_ptr ? nullptr : t.normal[i];
        }
        at += o->view_bytes[i];
    }
    return BGS_OK;
}

}  // namespace

namespace bgs {

FrameConsts frame_consts(const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
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
    fc.cov_pre = cloud->layout == CloudLayout::F16Cov ? 1u : 0u;
    memcpy(fc.aabb_min, uni->aabb_min, 12); memcpy(fc.aabb_max, uni->aabb_max, 12);
    static const float kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    fc.model_identity = memcmp(uni->transform, kIdentity, 64) == 0 ? 1u : 0u;   // (-0.0 entries take the general path)
    return fc;
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
        if (c->kg_grid == 0 || c->bin_grid == 0 || c->rs_per_sm == 0 || c->kg_scene_per_sm == 0) coop = 0;
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
    }
    cudaSetDevice(c->device);
    c->each_stream([](cudaStream_t& s, int) { if (s) cudaStreamSynchronize(s); });
    c->each_event([](cudaEvent_t& ev, bool) { if (ev) cudaEventDestroy(ev); });
    c->each_stream([](cudaStream_t& s, int) { if (s) cudaStreamDestroy(s); });
    if (c->h_ctr) cudaFreeHost(c->h_ctr);
    if (c->h_sticky) cudaFreeHost(c->h_sticky);
    if (c->h_word) cudaFreeHost(c->h_word);
    if (c->h_bounce) cudaFreeHost(c->h_bounce);
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

static bgs_status check_render(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                               const bgs_settings* st, const bgs_render_extras* ex, uint32_t out_format, bool want_aux,
                               bool temporal) {
    // not-ready inputs map to the reference's silent skip-frame (radix.rs:645-658, mod.rs:1533-1539)
    if (!cloud || !view || !uni || !st) return fail(c, BGS_NOT_READY, "render: cloud/view/uniform/settings not ready");
    TRY(enter_call(c, "render", cloud->device));   // (contexts of one GPU may share clouds)
    if (out_format > BGS_FORMAT_RGBA32F) return fail(c, BGS_EINVAL, "render: unknown out_format %u", out_format);
    if (st->radix_sort_depth_bits != 16 && st->radix_sort_depth_bits != 24 && st->radix_sort_depth_bits != 32)
        return fail(c, BGS_EINVAL, "render: radix_sort_depth_bits must be 16, 24 or 32");
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
    if (st->rasterize_mode == BGS_RASTERIZE_OPTICAL_FLOW) {
        if (!ex) return fail(c, BGS_EINVAL, "render: OpticalFlow needs the previous view (bgs_render_ex extras)");
        if (!(std::isfinite(ex->delta_time) && ex->delta_time > 0.0f))
            return fail(c, BGS_EINVAL, "render: OpticalFlow delta_time %g is not finite and > 0", (double)ex->delta_time);
        for (int i = 0; i < 16; ++i)
            if (!std::isfinite(ex->previous_clip_from_world[i]))
                return fail(c, BGS_EINVAL, "render: previous_clip_from_world[%d] is not finite", i);
    }
    if (st->draw_mode > BGS_DRAW_HIGHLIGHT_SELECTED) return fail(c, BGS_EINVAL, "render: bad draw_mode");
    if (cloud->layout == CloudLayout::F16Cov && (st->gaussian_mode != BGS_GAUSSIAN_3D || st->rasterize_mode == BGS_RASTERIZE_NORMAL || want_aux))
        return fail(c, BGS_EINVAL, "render: a precomputed-covariance cloud has no rotation / scale: Gaussian3d with Color, Depth or Position only");
    const int W = (int)view->viewport[2], H = (int)view->viewport[3];
    if (W <= 0 || H <= 0 || W > 65535 || H > 65535) return fail(c, BGS_EINVAL, "render: viewport %dx%d out of range", W, H);
    return BGS_OK;
}


// Enqueues one attempt at a frame: every launch of the plan, the counters' read-back and the copy-out.  A scene frame
// (render_entities_impl) runs key-gen, the depth range, the projection and the splat depths over its segment table; `cloud`
// is then its first cloud and fc its first segment's.
static bgs_status enqueue_frame(bgs_context* c, const bgs_cloud* cloud, const FrameConsts& fc, const ModeConsts* modes,
                                const TemporalConsts* tc, const FramePlan& p, const FrameOut& o, const bgs_scene_depth* zd,
                                const std::shared_ptr<const SceneFacts>& scene, const ViewTable* views) {
    const uint32_t n = scene ? scene->tab.n_total : cloud->n;
    // (a views frame: every view's tiles, one global tile id space)
    const uint32_t num_tiles = views ? views->tile0[views->v] : (uint32_t)fc.tiles_x * (uint32_t)fc.tiles_y;
    cudaStream_t q = c->stream;
    uint32_t launches = 0;
    if (scene) {
        const std::vector<const bgs_cloud*>& cl = scene->clouds;
        for (size_t j = 0; j < cl.size(); ++j)
            if (std::find(cl.begin(), cl.begin() + j, cl[j]) == cl.begin() + j) TRY(before_cloud_read(c, cl[j]));
    } else {
        TRY(before_cloud_read(c, cloud));
    }
    CU(c, cudaMemsetAsync(c->arena.p, 0, c->arena.bytes, q));   // counters, histograms, ranges: ~0.4 MB
    CU(c, cudaEventRecord(c->ev[0], q));
    // ---- stage 1: key-gen (+ stable compaction of the visible set)
    // compact mode: keys[0][slot], slot_ids[slot] = gaussian index, vals[0][slot] = slot (sort payload)
    // SORT_ALL    : keys[0][i], vals[0][i] = i (payload is the gaussian index itself)
    if (scene) {   // (scenes are compact frames)
        // key-gen gathers the culled ends for the Depth range when segment 0 is in Depth mode: when only some other
        // entity is, it reads a copy of the table whose segment 0 is
        SceneTable kt;
        const bool depth0 = p.depth_range && scene->tab.seg[0].fc.rasterize_mode != BGS_RASTERIZE_DEPTH;
        if (depth0) {
            kt = scene->tab;
            kt.seg[0].fc.rasterize_mode = BGS_RASTERIZE_DEPTH;
        }
        CU(c, launch_keygen_scene(depth0 ? kt : scene->tab, c->keys[1].p, c->keys[0].p, c->slot_ids.p, c->vals[0].p,
                                  c->kg_block_cnt, c->ctr, c->hist, p.depth_passes,
                                  std::min(p.kg_grid, (uint32_t)c->sm_count * c->kg_scene_per_sm), q));
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
        else if (scene) launch_depth_range_scene(scene->tab, c->vals[cur].p, c->slot_ids.p, c->ctr, q);
        else launch_depth_range(cloud->pos, n, c->vals[cur].p, p.by_slot ? c->slot_ids.p : nullptr, c->ctr, fc, q);
        ++launches;
    }
    CU(c, cudaEventRecord(c->ev_p0, ps));
    bool scene_3d = false;   // a scene lists a non-4D cloud (whose splat depths splat_depth_scene writes)
    if (scene) {   // one launch per projection group: each segment with its own settings and num_classes
        for (size_t i = 0; i < scene->groups.size(); ++i) {
            const uint32_t g = scene->groups[i];
            if (g == PROJECT_GROUP_4D) {   // (also writes the 4D segments' splat depths, from the moved positions)
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
    ZTestArgs zt;
    if ((zd || o.pick) && scene_3d) {
        launch_splat_depth_scene(scene->tab, c->slot_ids.p, c->ctr, c->splat_depth.p, p.n_hint, c->sm_count, ps);
        ++launches;
    } else if (zd && !tc && !scene) {
        launch_splat_depth(cloud->pos, p.by_slot ? c->slot_ids.p : c->vals[cur].p, p.by_slot ? 1 : 0, c->ctr, fc,
                           c->splat_depth.p, p.n_hint, c->sm_count, ps);
        ++launches;
    }
    if (zd) { zt.splat_d = c->splat_depth.p; zt.scene = zd->depth; zt.pitch = (size_t)zd->pitch_bytes; }
    if (o.pick) zt.splat_d = c->splat_depth.p;
    if (p.overlap) {
        CU(c, cudaEventRecord(c->ev_join, c->stream2));
        CU(c, cudaStreamWaitEvent(q, c->ev_join, 0));
    }
    CU(c, cudaEventRecord(c->ev[3], q));
    if (p.raster_mode >= 3) {   // a mixed-geometry frame: each record's blend kind, for the blend
        launch_segment_kinds(scene->kinds, c->slot_ids.p, c->ctr, c->kinds.p, p.n_hint, c->sm_count, q);
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
        if (r + 1 == p.rounds) {
            // (chunked frames: the earlier rounds' blends are accounted to stage 4)
            CU(c, cudaEventRecord(c->ev[4], q));
            if (o.slot >= 0 && c->copy_pending[o.slot]) CU(c, cudaStreamWaitEvent(q, c->ev_copied[o.slot], 0));   // target free again
        }
        if (p.rounds == 1) {
            // the blend runs on the LOW-priority stream; the render stream resumes once it is done
            CU(c, cudaEventRecord(c->ev_front, q));
            CU(c, cudaStreamWaitEvent(c->stream_r, c->ev_front, 0));
            if (o.pick)
                launch_raster_pick(p.raster_mode, c->recs.p, c->extra.p, c->pvals[pcur].p, rng, fc.Wi, fc.Hi, fc.tiles_x,
                                   fc.tiles_y, o.rgba, o.raster_format, &c->ctr->truncated, zt, c->kinds.p, p.box,
                                   PickArgs{o.pick, c->slot_ids.p, scene->kinds}, c->stream_r);
            else if (views)
                launch_raster_views(p.raster_mode, c->recs.p, c->extra.p, c->pvals[pcur].p, rng, o.raster_format,
                                    &c->ctr->truncated, zt.splat_d, c->kinds.p, p.box, *views, c->stream_r,
                                    fc.aux ? c->aux.p : nullptr);
            else
                launch_raster(p.raster_mode, p.large_fp, c->recs.p, c->extra.p, c->pvals[pcur].p, rng, fc.Wi, fc.Hi, fc.tiles_x,
                              fc.tiles_y, o.rgba, o.raster_format, fc.aux ? c->aux.p : nullptr, o.depth, o.normal,
                              &c->ctr->truncated, zt, c->stream_r, c->kinds.p, p.box);
            CU(c, cudaEventRecord(c->ev_rdone, c->stream_r));
            CU(c, cudaStreamWaitEvent(q, c->ev_rdone, 0));
        } else
            launch_raster_round(c->recs.p, c->pvals[pcur].p, rng, fc.Wi, fc.Hi, fc.tiles_x, fc.tiles_y, o.rgba, o.raster_format,
                                c->state.p, c->tile_done, &c->ctr->tiles_done, &c->ctr->truncated, r == 0, r + 1 == p.rounds, zt,
                                q);
        ++launches;
    }
    c->pair_result = pcur;
    CU(c, cudaEventRecord(c->ev[5], q));
    CU(c, cudaEventRecord(c->ev_done, q));
    CU(c, cudaMemcpyAsync(c->h_ctr, c->ctr, sizeof(FrameCounters), cudaMemcpyDeviceToHost, q));
    CU(c, cudaMemcpyAsync(c->h_sticky, c->d_sticky, 4, cudaMemcpyDeviceToHost, q));
    if (o.slot >= 0) CU(c, cudaEventRecord(c->ev_raster[o.slot], q));
    // a views frame to host memory: each view's frames to its own host targets
    auto copy_views = [&](cudaStream_t s) -> bgs_status {
        for (uint32_t i = 0; i < o.views; ++i) {
            CU(c, cudaMemcpyAsync(o.view_host[i], o.view_rgba[i], o.view_bytes[i], cudaMemcpyDeviceToHost, s));
            if (o.view_host_depth[i]) {
                CU(c, cudaMemcpyAsync(o.view_host_depth[i], o.view_depth[i], o.view_bytes[i], cudaMemcpyDeviceToHost, s));
                CU(c, cudaMemcpyAsync(o.view_host_normal[i], o.view_normal[i], o.view_bytes[i], cudaMemcpyDeviceToHost, s));
            }
        }
        return BGS_OK;
    };
    const bool views_to_host = o.views > 0 && o.view_host[0] != nullptr;
    if (o.slot >= 0 && (o.host_rgba || views_to_host)) {
        CU(c, cudaStreamWaitEvent(c->stream_copy, c->ev_raster[o.slot], 0));
        if (views_to_host) TRY(copy_views(c->stream_copy));
        else CU(c, cudaMemcpyAsync(o.host_rgba, o.rgba, o.bytes, cudaMemcpyDeviceToHost, c->stream_copy));
        CU(c, cudaEventRecord(c->ev_copied[o.slot], c->stream_copy));
        c->copy_pending[o.slot] = true;
    } else if (views_to_host) {
        TRY(copy_views(q));
    } else if (o.host_rgba) {
        CU(c, cudaMemcpyAsync(o.host_rgba, o.rgba, o.bytes, cudaMemcpyDeviceToHost, q));
        if (o.host_depth) {
            CU(c, cudaMemcpyAsync(o.host_depth, o.depth, o.bytes, cudaMemcpyDeviceToHost, q));
            CU(c, cudaMemcpyAsync(o.host_normal, o.normal, o.bytes, cudaMemcpyDeviceToHost, q));
        }
        if (o.host_pick)
            CU(c, cudaMemcpyAsync(o.host_pick, o.pick, (size_t)fc.Wi * fc.Hi * sizeof(bgs_pick), cudaMemcpyDeviceToHost, q));
    }
    c->pend = {cloud, n, fc, !p.by_slot, p.by_slot, p.rounds, views ? (int)num_tiles : fc.tiles_x, views ? 1 : fc.tiles_y, fc.Wi,
               fc.Hi, o.rgba, zd != nullptr || o.pick != nullptr, scene};
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
                              const bgs_settings* st, const bgs_render_extras* ex, void* out_rgba, uint32_t out_format,
                              int out_is_device_ptr, bool want_aux, void* out_depth, void* out_normal,
                              const bgs_scene_depth* zd = nullptr, const TemporalConsts* tc = nullptr,
                              const std::shared_ptr<const SceneFacts>& scene = nullptr, const ViewTargets* view_targets = nullptr,
                              void* out_pick = nullptr) {
    if (!c) return BGS_EINVAL;
    if (!scene) TRY(check_render(c, cloud, view, uni, st, ex, out_format, want_aux, tc != nullptr));   // (scenes: per cloud, before)
    if (zd) TRY(check_scene_depth(c, zd, view));
    if (c->async_pending && !(st->flags & BGS_FLAG_ASYNC)) {
        // a synchronous render after queued frames completes them first; their failure (including an overflowed
        // pair list = BGS_NOT_READY) is the caller's to see, so this frame is not rendered on top of it
        TRY(bgs_sync(c));
    }
    const FrameConsts fc = scene ? scene->tab.seg[0].fc : frame_consts(cloud, view, uni, st, want_aux);
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
    if (views) TRY(frame_out_views(c, st, out_format, scene->views, *view_targets, out_is_device_ptr, &o));
    else TRY(frame_out(c, st, out_format, (size_t)fc.Wi * fc.Hi * format_bpp(out_format), out_rgba, out_is_device_ptr, want_aux,
                       out_depth, out_normal, &o));
    if (out_pick && out_is_device_ptr) {
        o.pick = static_cast<uint4*>(out_pick);
    } else if (out_pick) {
        TRY(c->pick_frame.grow(c, (size_t)fc.Wi * fc.Hi * sizeof(bgs_pick), false));
        o.pick = c->pick_frame.p;
        o.host_pick = out_pick;
    }
    ViewTable vt = {};
    if (views) {
        vt = scene->views;
        for (uint32_t i = 0; i < vt.v; ++i) {
            vt.out[i] = o.view_rgba[i];
            vt.out_depth[i] = o.view_depth[i];
            vt.out_normal[i] = o.view_normal[i];
        }
    }
    for (int attempt = 0; attempt < 4; ++attempt) {
        FramePlan p = plan_frame(c, st, want_aux, num_tiles, n);   // (each attempt: the pair hints read cap_pairs)
        if (scene) {   // (st plans it as an aabb frame or an overlay one: one round)
            p.raster_mode = scene->raster_mode;
            p.box = scene->box;
        }
        if (p.raster_mode == 2 || p.raster_mode == 4) TRY(c->extra.grow(c, (size_t)c->cap_n * 64, false));
        if (p.raster_mode >= 3) TRY(c->kinds.grow(c, (size_t)c->cap_n, false));
        if (want_aux) TRY(c->aux.grow(c, (size_t)c->cap_n * 32, false));
        if (zd || o.pick) TRY(c->splat_depth.grow(c, (size_t)c->cap_n * 4, false));
        if (p.rounds > 1) TRY(c->state.grow(c, (size_t)num_tiles * 256 * sizeof(float4), false));
        TRY(ensure_arena(c, num_tiles));
        TRY(ensure_status(c, c->status_depth, c->status_n, n));
        TRY(ensure_status(c, c->status_pairs, c->status_np, c->cap_pairs));
        TRY(enqueue_frame(c, cloud, fc, modes, tc, p, o, zd, scene, views ? &vt : nullptr));
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
    return render_impl(c, cloud, view, uni, st, ex, out_rgba, out_format, out_is_device_ptr, false, nullptr, nullptr);
}

bgs_status bgs_render_depth_test(bgs_context* c, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni,
                                 const bgs_settings* st, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                 void* out_rgba, uint32_t out_format, int out_is_device_ptr) {
    return render_impl(c, cloud, view, uni, st, ex, out_rgba, out_format, out_is_device_ptr, false, nullptr, nullptr, depth);
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
    return render_impl(c, cloud, view, uni, st, ex, out_rgba, out_format, out_is_device_ptr, false, nullptr, nullptr, depth, &tc);
}

// the refusals every scene call makes of its list before reading it: k, SORT_ALL and NULL clouds
static bgs_status check_scene_list(bgs_context* c, const char* call, const bgs_cloud* const* clouds, uint32_t k,
                                   const bgs_settings* frame) {
    if (k == 0 || k > BGS_SCENE_MAX_CLOUDS) return fail(c, BGS_EINVAL, "%s: k = %u is not in 1..%d", call, k, BGS_SCENE_MAX_CLOUDS);
    if (frame->flags & BGS_FLAG_SORT_ALL) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_SORT_ALL is not supported", call);
    for (uint32_t j = 0; j < k; ++j)
        if (!clouds[j]) return fail(c, BGS_EINVAL, "%s: clouds[%u] is NULL", call, j);
    return BGS_OK;
}

// the blend kind of an entity's records (raster.cu): 0 = quad-uv, 1 = conic (3DGS and 4D with aabb), 2 = surfel
static int blend_kind(const bgs_entity_settings& e) { return !e.aabb ? 0 : (e.gaussian_mode == BGS_GAUSSIAN_2D ? 2 : 1); }

// Every scene frame: k entities, each checked as its single-cloud call (bgs_render_depth_test, or bgs_render_4d for a
// Gaussian4d cloud when with_4d) with its own settings, num_classes and window, drawn into one depth-sorted frame.
// entity_flags: each entity's BGS_ENTITY_* bits (NULL: none).  The list has passed check_scene_list.  want_aux
// (bgs_render_entities_aux): every segment also projects its Depth and Normal colours, blended into out_depth / out_normal.
// nv > 1 (bgs_render_views or, with want_aux, bgs_render_views_aux, which have checked nv, the targets and the entities'
// modes): the k entities seen from each of the nv views (depth: nv buffers, or NULL), segment i k + j entity j from view i,
// view i's frames into view_targets' entries i.
static bgs_status render_entities_impl(bgs_context* c, const char* call, bool with_4d, const bgs_cloud* const* clouds,
                                       const bgs_cloud_uniform* unis, const bgs_entity_settings* ents,
                                       const uint32_t* entity_flags, uint32_t k, const bgs_view* view,
                                       const bgs_settings* frame, const bgs_render_extras* ex, const bgs_scene_depth* depth,
                                       void* out_rgba, uint32_t out_format, int out_is_device_ptr, bool want_aux = false,
                                       void* out_depth = nullptr, void* out_normal = nullptr, uint32_t nv = 1,
                                       const ViewTargets* view_targets = nullptr, void* out_pick = nullptr) {
    // each entity's bounding-box overlay: its own bit, or the frame's flag for every entity
    auto box_of = [&](uint32_t j) {
        return (frame->flags & BGS_FLAG_VISUALIZE_BOUNDING_BOX) != 0 ||
               (entity_flags && (entity_flags[j] & BGS_ENTITY_VISUALIZE_BOUNDING_BOX) != 0);
    };
    // entity j as its single-cloud call: its settings with the frame's sort bits and flags, its num_classes and window
    std::vector<bgs_settings> st(k);
    auto scene = std::make_shared<SceneFacts>();
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
            TRY(check_render(c, clouds[j], &view[i], &unis[j], &chk,
                             ex || e.rasterize_mode == BGS_RASTERIZE_CLASSIFICATION ? &ej : nullptr, out_format, false, is4));
        if (is4) TRY(temporal_consts(c, call, unis[j].time, e.window.time_start, e.window.time_stop, scene->times.t[j]));
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
    SceneTable& tab = scene->tab;
    memset(&tab, 0, sizeof(tab));
    tab.k = k * nv;
    tab.n_total = (uint32_t)total;
    scene->kinds.k = k * nv;
    uint32_t offset = 0;
    bool box_all = true;
    for (uint32_t i = 0; i < nv; ++i)
        for (uint32_t j = 0; j < k; ++j) {
            const uint32_t sj = i * k + j;   // entity j seen from view i
            const bgs_cloud* cl = clouds[j];
            const uint32_t rm = st[j].rasterize_mode;
            SceneSeg& sg = tab.seg[sj];
            sg.fc = frame_consts(cl, &view[i], &unis[j], &st[j], want_aux);
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
            scene->times.t[sj] = scene->times.t[j];
            scene->classes.n[sj] = ents[j].num_classes;
            scene->kinds.offset[sj] = offset;
            scene->kinds.kind[sj] = (uint32_t)blend_kind(ents[j]) | (box_of(j) ? BOX_KIND : 0u);
            scene->box = scene->box || box_of(j);
            box_all = box_all && box_of(j);
            offset += cl->n;
            scene->clouds.push_back(cl);
        }
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
    if (nv > 1 || out_pick) sf.flags = (sf.flags & ~(uint32_t)BGS_FLAG_CHUNKS) | BGS_FLAG_NO_CHUNKS;   // (one round)
    return render_impl(c, clouds[0], view, &unis[0], &sf, ex, out_rgba, out_format, out_is_device_ptr, want_aux, out_depth,
                       out_normal, depth, nullptr, scene, view_targets, out_pick);
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
    return render_entities_impl(c, call, with_4d, clouds, unis, ents.data(), nullptr, k, view, st, ex, depth, out_rgba,
                                out_format, out_is_device_ptr);
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
                                      const uint32_t* entity_flags, uint32_t k, const bgs_view* view, const bgs_settings* frame) {
    if (!clouds || !unis || !ents || !view || !frame)
        return fail(c, BGS_NOT_READY, "%s: clouds/uniforms/entities/view/settings not ready", call);
    TRY(check_scene_list(c, call, clouds, k, frame));
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
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth, out_rgba, out_format,
                                out_is_device_ptr);
}

// bgs_render_entities_ex's frame and, in the same pass, its Depth and Normal frames (include/bgs.h): the refusals of
// bgs_render_entities_ex, then those of the aux frames
bgs_status bgs_render_entities_aux(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                   const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k,
                                   const bgs_view* view, const bgs_settings* frame, const bgs_render_extras* ex,
                                   const bgs_scene_depth* depth, void* out_rgba, void* out_depth, void* out_normal,
                                   uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_entities_aux";
    if (!c) return BGS_EINVAL;
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, view, frame));
    if (!out_rgba || !out_depth || !out_normal) return fail(c, BGS_EINVAL, "%s: the three output frames are required", call);
    if (frame->flags & BGS_FLAG_ASYNC) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_ASYNC is not supported", call);
    for (uint32_t j = 0; j < k; ++j) {
        // (a 4D cloud has no Normal colour; a covariance cloud no rotation; Velocity changes which splats draw, and how)
        if (is_4d(clouds[j]->layout)) return fail(c, BGS_EINVAL, "%s: clouds[%u] is a Gaussian4d cloud", call, j);
        if (clouds[j]->layout == CloudLayout::F16Cov)
            return fail(c, BGS_EINVAL, "%s: clouds[%u] is a precomputed-covariance cloud (no rotation for the normal)", call, j);
        if (ents[j].rasterize_mode == BGS_RASTERIZE_VELOCITY)
            return fail(c, BGS_EINVAL, "%s: entities[%u] is in Velocity mode", call, j);
    }
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth, out_rgba, out_format,
                                out_is_device_ptr, true, out_depth, out_normal);
}

// bgs_render_entities_ex's frame and, from the same blend, its pick frame (include/bgs.h): the refusals of
// bgs_render_entities_ex, then those of the pick target
bgs_status bgs_render_entities_pick(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                    const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k,
                                    const bgs_view* view, const bgs_settings* frame, const bgs_render_extras* ex,
                                    const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format, int out_is_device_ptr,
                                    void* out_pick) {
    const char* call = "render_entities_pick";
    if (!c) return BGS_EINVAL;
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, view, frame));
    if (!out_pick) return fail(c, BGS_EINVAL, "%s: out_pick is NULL", call);
    if (out_is_device_ptr && reinterpret_cast<uintptr_t>(out_pick) % sizeof(bgs_pick) != 0)
        return fail(c, BGS_EINVAL, "%s: device pick target %p is not aligned to its 16-byte records", call, out_pick);
    if (frame->flags & BGS_FLAG_ASYNC) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_ASYNC is not supported", call);
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, view, frame, ex, depth, out_rgba, out_format,
                                out_is_device_ptr, false, nullptr, nullptr, 1, nullptr, out_pick);
}

// bgs_render_entities_ex of each of v views in one frame (include/bgs.h): the refusals of bgs_render_entities_ex (each view
// checked as its own call), then those of the views frame; one view is bgs_render_entities_ex itself
bgs_status bgs_render_views(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                            const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* views,
                            uint32_t v, const bgs_settings* frame, const bgs_scene_depth* depths, void* const* out_rgba,
                            uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_views";
    if (!c) return BGS_EINVAL;
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, views, frame));
    if (v == 0) return fail(c, BGS_EINVAL, "%s: v = 0 views", call);
    if ((uint64_t)v * k > BGS_SCENE_MAX_CLOUDS)
        return fail(c, BGS_EINVAL, "%s: v x k = %u x %u segments, at most %d", call, v, k, BGS_SCENE_MAX_CLOUDS);
    if (!out_rgba) return fail(c, BGS_EINVAL, "%s: out_rgba is NULL", call);
    const size_t bpp = format_bpp(out_format);
    for (uint32_t i = 0; i < v; ++i) {
        if (!out_rgba[i]) return fail(c, BGS_EINVAL, "%s: out_rgba[%u] is NULL", call, i);
        if (out_is_device_ptr && reinterpret_cast<uintptr_t>(out_rgba[i]) % bpp != 0)
            return fail(c, BGS_EINVAL, "%s: device target out_rgba[%u] = %p is not aligned to its %zu-byte pixels", call, i,
                        out_rgba[i], bpp);
    }
    for (uint32_t j = 0; j < k; ++j) {
        // (a Depth entity's colour range is the frame's sorted list; OpticalFlow has one previous view per frame)
        if (ents[j].rasterize_mode == BGS_RASTERIZE_DEPTH) return fail(c, BGS_EINVAL, "%s: entities[%u] is in Depth mode", call, j);
        if (ents[j].rasterize_mode == BGS_RASTERIZE_OPTICAL_FLOW)
            return fail(c, BGS_EINVAL, "%s: entities[%u] is in OpticalFlow mode", call, j);
    }
    if ((frame->flags & BGS_FLAG_BLEND_OVER_TARGET) && !out_is_device_ptr)
        return fail(c, BGS_EINVAL, "%s: BGS_FLAG_BLEND_OVER_TARGET takes device targets", call);
    if (v == 1)
        return bgs_render_entities_ex(c, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, out_rgba[0], out_format,
                                      out_is_device_ptr);
    const ViewTargets targets{out_rgba, nullptr, nullptr};
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, nullptr,
                                out_format, out_is_device_ptr, false, nullptr, nullptr, v, &targets);
}

// bgs_render_entities_aux of each of v views in one frame (include/bgs.h): the refusals of bgs_render_entities_aux and of
// bgs_render_views but the Depth one, then those of its three target arrays; one view is bgs_render_entities_aux itself
bgs_status bgs_render_views_aux(bgs_context* c, const bgs_cloud* const* clouds, const bgs_cloud_uniform* unis,
                                const bgs_entity_settings* ents, const uint32_t* entity_flags, uint32_t k, const bgs_view* views,
                                uint32_t v, const bgs_settings* frame, const bgs_scene_depth* depths, void* const* out_rgba,
                                void* const* out_depth, void* const* out_normal, uint32_t out_format, int out_is_device_ptr) {
    const char* call = "render_views_aux";
    if (!c) return BGS_EINVAL;
    TRY(check_entities_call(c, call, clouds, unis, ents, entity_flags, k, views, frame));
    if (v == 0) return fail(c, BGS_EINVAL, "%s: v = 0 views", call);
    if ((uint64_t)v * k > BGS_SCENE_MAX_CLOUDS)
        return fail(c, BGS_EINVAL, "%s: v x k = %u x %u segments, at most %d", call, v, k, BGS_SCENE_MAX_CLOUDS);
    const size_t bpp = format_bpp(out_format);
    const char* names[3] = {"out_rgba", "out_depth", "out_normal"};
    void* const* arrays[3] = {out_rgba, out_depth, out_normal};
    for (int a = 0; a < 3; ++a) {
        if (!arrays[a]) return fail(c, BGS_EINVAL, "%s: %s is NULL", call, names[a]);
        for (uint32_t i = 0; i < v; ++i) {
            if (!arrays[a][i]) return fail(c, BGS_EINVAL, "%s: %s[%u] is NULL", call, names[a], i);
            if (out_is_device_ptr && reinterpret_cast<uintptr_t>(arrays[a][i]) % bpp != 0)
                return fail(c, BGS_EINVAL, "%s: device target %s[%u] = %p is not aligned to its %zu-byte pixels", call, names[a],
                            i, arrays[a][i], bpp);
        }
    }
    if (frame->flags & BGS_FLAG_ASYNC) return fail(c, BGS_EINVAL, "%s: BGS_FLAG_ASYNC is not supported", call);
    for (uint32_t j = 0; j < k; ++j) {
        // (bgs_render_entities_aux's refusals; OpticalFlow has one previous view per frame)
        if (is_4d(clouds[j]->layout)) return fail(c, BGS_EINVAL, "%s: clouds[%u] is a Gaussian4d cloud", call, j);
        if (clouds[j]->layout == CloudLayout::F16Cov)
            return fail(c, BGS_EINVAL, "%s: clouds[%u] is a precomputed-covariance cloud (no rotation for the normal)", call, j);
        if (ents[j].rasterize_mode == BGS_RASTERIZE_VELOCITY)
            return fail(c, BGS_EINVAL, "%s: entities[%u] is in Velocity mode", call, j);
        if (ents[j].rasterize_mode == BGS_RASTERIZE_OPTICAL_FLOW)
            return fail(c, BGS_EINVAL, "%s: entities[%u] is in OpticalFlow mode", call, j);
    }
    if ((frame->flags & BGS_FLAG_BLEND_OVER_TARGET) && !out_is_device_ptr)
        return fail(c, BGS_EINVAL, "%s: BGS_FLAG_BLEND_OVER_TARGET takes device targets", call);
    if (v == 1)
        return bgs_render_entities_aux(c, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, out_rgba[0],
                                       out_depth[0], out_normal[0], out_format, out_is_device_ptr);
    const ViewTargets targets{out_rgba, out_depth, out_normal};
    return render_entities_impl(c, call, true, clouds, unis, ents, entity_flags, k, views, frame, nullptr, depths, nullptr,
                                out_format, out_is_device_ptr, true, nullptr, nullptr, v, &targets);
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
    return render_impl(c, cloud, view, uni, st, nullptr, out_rgba, out_format, out_is_device_ptr, true, out_depth, out_normal);
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
        if (c->last.scene) launch_culled_flags_scene(c->last.scene->tab, flags, c->stream);
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
