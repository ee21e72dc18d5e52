// host.cuh -- what libbgs's two host halves share: api.cu (contexts, the per-view frame, the debug hooks) and cloud.cu
// (the calls on a resident cloud).  The objects behind include/bgs.h's handles, error reporting, the context registry,
// the order of a cloud's accesses, and the frame scratch that the selections borrow.
#pragma once
#include <algorithm>
#include <array>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "launch.cuh"

namespace bgs {

// A grow-only device buffer.  grow() replaces a buffer smaller than `want` bytes by one of exactly `want` bytes, zeroed
// on the render stream when asked; a failed grow leaves it empty.  Its owner (the context) releases it on destruction.
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

// Regions of one byte buffer, each starting on a 256 B boundary: add() returns a region's offset, `end` is one past
// the last region and padded() that rounded up to 256 B.
struct Layout {
    size_t end = 0;
    static size_t align_up(size_t v) { return (v + 255) / 256 * 256; }
    size_t add(size_t bytes) { const size_t o = align_up(end); end = o + bytes; return o; }
    size_t padded() const { return align_up(end); }
};

}  // namespace bgs

using namespace bgs;

struct bgs_cloud {
    int device;       // the CUDA device the planes live on
    uint32_t n;
    CloudLayout layout;
    uint32_t sh_degree;         // 0..3 (include/bgs.h); 3 for every cloud of the calls without _sh, 4D clouds included
    float4* pos = nullptr;      // the position plane and the gaussian-major blocks (cloud_layout.cuh)
    void* blocks = nullptr;
    // enqueued writes (particle steps): ev_write marks the last one, on whichever context's stream it was queued; every
    // later reader or writer waits for it on the device.  Created by the first step; `stepped` is set once it exists,
    // so a cloud that is never stepped costs its frames nothing
    cudaEvent_t ev_write = nullptr;
    std::atomic<bool> stepped{false};
    CloudView view() const { return {pos, static_cast<uint4*>(blocks), chunks(layout, sh_degree)}; }
};

// A ParticleBehaviors asset resident on one GPU: count 64 B records (bgs_particle_behavior), read and written by the step
struct bgs_particles {
    int device;
    uint32_t count;
    int64_t max_index;            // largest active gaussian index (-1: none is active)
    void* d = nullptr;            // count * 64 B
    cudaEvent_t ev_write = nullptr;   // the last step of these behaviours (recorded on the stepping context's stream)
};

// One generation of a bgs_entity_list's device arrays, cap entities each: the compact records, the segment table's
// offset, time, num_classes and kind arrays (kinds_box: the kinds with BOX_KIND set, for frames with the frame-wide
// overlay), and the segments the expansion writes once per frame.  A frame holds the generation it reads (SceneFacts), so
// an edit writes the list's current generation in place only when no frame holds it (api.cu: list_writable).
struct ListTable {
    uint32_t cap = 0;
    DevBuf<uint8_t> mem;
    EntityListArrays a = {};
    SceneSeg* seg = nullptr;
};

// A scene frame (bgs_render_scene, _scene_4d, _entities): its segment table (what its kernels and the culled-flags hook
// read), its 4D segments' times, the clouds it lists (clouds[j] is segment j's; a cloud may be listed more than once),
// its distinct projection groups (project_group, plus ENTITY_MODES for the Classification / OpticalFlow / Velocity colour
// kernel, or PROJECT_GROUP_4D) with whether one of each group's segments reads the SH coefficients, the segments'
// num_classes, the blend (raster.cu's mode: 0..2 when every splat has one kind, else 3 / 4 with `kinds`), and whether
// some entity draws its bounding boxes (kinds' BOX_KIND bits say which, on mixed frames; on the others every entity does)
struct SceneFacts {
    SceneTable tab;
    SceneTimes times = {};
    std::vector<const bgs_cloud*> clouds;
    std::vector<const bgs_cloud*> distinct;   // the clouds listed, each once (sorted by address)
    std::vector<uint32_t> groups;
    std::vector<uint32_t> need_sh;   // per entry of groups
    SceneClasses classes = {};
    int raster_mode = 0;
    SegmentKinds kinds = {};
    bool box = false;
    // a views frame (bgs_render_views, _views_aux, views.v > 1): the table has views.v x k segments, segment i k + j entity j
    // seen from view i; the views' tile geometry and depth buffers (their targets are the frame's, filled in when it is
    // enqueued)
    ViewTable views = {};
    // a bgs_render_entities_many frame: the segments, times, num_classes and kinds are in the device table dtab (tab holds
    // N and segment 0 alone), which enqueue_frame copies from the pinned staging h_tab (tab_bytes) of the context's table
    // slot `slot` (bgs_context::many)
    bool many = false;
    SceneTableDev dtab = {};
    const void* h_tab = nullptr;
    size_t tab_bytes = 0;
    int slot = 0;
    // a bgs_render_entity_list frame: dtab is generation `list_tab` of the list, whose segments the frame's first launch
    // expands from its records and the view (radix_sort_depth_bits: the frame's)
    const bgs_entity_list* list = nullptr;
    std::shared_ptr<ListTable> list_tab;
    bgs_view list_view = {};
    uint32_t list_depth_bits = 0;
};

// What the host knows of a frame it has enqueued: the context keeps the last one enqueued (`pend`) and, once its
// counters are back, the last one completed (`last`, what the debug hooks read).
struct FrameFacts {
    const bgs_cloud* cloud = nullptr;   // (nulled if the cloud is destroyed meanwhile; a scene frame's first cloud)
    uint32_t n = 0;                     // gaussians in the cloud, or the scene's N (a snapshot: the cloud may be gone by the time it is read)
    FrameConsts fc = {};
    bool sort_all = false;
    bool by_slot = false;               // records indexed by compact slot (else by front-to-back rank)
    int rounds = 1;                     // binning rounds
    int tiles_x = 0, tiles_y = 0, W = 0, H = 0;   // (a views frame: every view's tiles x 1, view 0's W x H)
    const void* target = nullptr;       // the device frame the blend wrote
    bool depth_tested = false;          // a depth buffer or a pick frame (bgs_render_entities_pick): splat_depth holds the splats' d
    std::shared_ptr<const SceneFacts> scene;   // bgs_render_scene frames only (nulled with `cloud`)
    bool reads(const bgs_cloud* cl) const {
        if (cloud == cl) return true;
        return scene && std::binary_search(scene->distinct.begin(), scene->distinct.end(), cl);
    }
    void forget() { cloud = nullptr; scene.reset(); }
};

struct bgs_context {
    int device = 0;
    int sm_count = 132;
    uint32_t kg_grid = 0, bin_grid = 0;   // co-resident grid sizes of the cooperative kernels (synchronous frames: latency)
    uint32_t kg_grid_async = 0, bin_grid_async = 0;   // ... of queued (BGS_FLAG_ASYNC) frames: 1 CTA per SM.  A latency-bound
                                          // cooperative grid holds its registers while it waits; with several frames in flight
                                          // a smaller grid leaves that room to the other frames' issue-bound blend
    int rs_per_sm = 0;                    // co-resident radix-sort CTAs per SM (radix.cu)
    uint32_t kg_scene_per_sm = 0;         // co-resident CTAs per SM of bgs_render_scene's key-gen (keygen.cu)
    uint32_t kg_many_per_sm = 0;          // ... of bgs_render_entities_many's
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
    DevBuf<float> splat_depth;        // 1 float per record: the splat depths d of depth-tested frames (allocated on first use)
    DevBuf<unsigned char> kinds;      // 1 byte per record: the blend kind of a mixed-geometry frame's splats (first use)
    DevBuf<void> frame_aux[2];        // depth / normal frames when an aux frame delivers to host memory (views: every view's)
    DevBuf<uint4> pick_frame;         // the pick frame when bgs_render_entities_pick delivers to host memory
    DevBuf<float4> sub_frames;        // bgs_render_shutter: each sample's raw (C, T) per pixel, s x W x H (grow-only)
    // scratch sized by the pair capacity (grow-only; cap_pairs pairs)
    uint32_t cap_pairs = 0;
    DevBuf<uint32_t> pkeys[2], pvals[2];
    DevBuf<float4> state;             // per-pixel blend state between rounds (tile-major), tiles * 256 * 16 B
    // zeroed-per-frame arena: counters | view ranges | hist | keygen CTA counts | bin CTA counts | ranges | done bytes
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
    // bgs_cloud_select_in_view's own scratch: its count word | a host mask's device copy
    DevBuf<uint8_t> view_select;
    // bgs_cloud_bounds' own words (transform.cu: launch_bounds)
    DevBuf<uint32_t> bounds_words;
    bool async_pending = false;        // a BGS_FLAG_ASYNC frame has been enqueued and not yet completed
    bool step_pending = false;         // a particle step has been enqueued since the last bgs_sync
    // an interpolation (a queued write that reads other clouds) has been enqueued since the last bgs_sync: ev_done
    // marks it, and the synchronous writers and bgs_cloud_destroy drain this context (set and read under the registry
    // lock; cleared by bgs_sync)
    std::atomic<bool> reads_pending{false};
    FrameCounters* ctr = nullptr;
    uint32_t* hist = nullptr;          // [8 + 4 * MAX_CHUNKS][256]: depth passes 0..3, pair passes 4..7 (round 0), 8 + 4r.. (round r)
    uint32_t* kg_block_cnt = nullptr;  // [kg_grid]: keygen_coop's per-CTA visible counts
    uint32_t* bin_block_cnt = nullptr; // [bin_grid][3]: bin_emit_coop's per-CTA pair / medium / large counts
    uint2* ranges = nullptr;           // per tile (~start, end) into the sorted pair list (0, 0 = empty)
    ViewRanges* view_ranges = nullptr; // bgs_render_views_aux: each view's Depth range
    unsigned char* tile_done = nullptr;   // per tile: saturated (chunked frames)
    // async frames delivered to host memory alternate the two frames so frame k's D2H copy (copy stream) overlaps
    // frame k+1's kernels
    DevBuf<void> frames[2];
    int frame_toggle = 0;              // the frame the next queued call that does not blend over takes
    int frame_last = 0;                // the frame the last call rendering into the library's frames wrote (blend-over's target)
    bool copy_pending[2] = {false, false};
    FrameCounters* h_ctr = nullptr;    // pinned
    float* cutoff_tab = nullptr;       // adaptive cutoff of every f16 opacity value (project.cu)
    // largest n_pairs_needed of ANY frame since the last bgs_sync / synchronous render (device word outside the
    // per-frame arena + its pinned copy): a queued async frame that overflowed the pair buffer is never missed
    uint32_t* d_sticky = nullptr;
    uint32_t* h_sticky = nullptr;
    uint32_t* h_word = nullptr;        // pinned: the one word a cloud call reads back (read_word)
    // bgs_cloud_download_*'s two pinned bounce buffers (2 x 30 MB, allocated by the first download, kept until the
    // context goes): one chunk's planes each, so the host's copy of one chunk overlaps the device-to-host copy of the next
    uint8_t* h_bounce = nullptr;

    // bgs_render_entities_many's segment tables: two slots, each a pinned staging buffer, its device copy (both grow-only)
    // and the event recorded after the last frame that read it.  A frame takes the slot the last one enqueued did not
    // (many_last), once that slot's frame has completed, so neither a queued frame's table nor the one the debug hooks of
    // the last frame read is overwritten.
    struct ManySlot {
        uint8_t* host = nullptr;
        size_t host_bytes = 0;
        DevBuf<uint8_t> dev;
        cudaEvent_t ev = nullptr;
        bool used = false;
    };
    ManySlot many[2];
    int many_last = 1;

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
                               &ev_copied[0], &ev_copied[1], &many[0].ev, &many[1].ev})
            f(*e, false);
    }
};

// An entity list resident on one context (bgs_entity_list): per entity what the host needs of it (x), and counters over
// the entities, kept by every edit, from which a frame takes its facts without a pass over the list.
struct ListEntity {
    const bgs_cloud* cloud;      // NULL once the cloud is destroyed (the entity is detached)
    bgs_cloud_uniform uni;       // as last given by the host (a transform set from device memory is not read back)
    bgs_entity_settings e;
    uint32_t flags;              // BGS_ENTITY_*
    uint32_t n, group, offset;   // the cloud's gaussians, the projection group, the first global index
    bool sh, is4;                // the group's launch reads SH coefficients for it; a Gaussian4d cloud
};
struct bgs_entity_list {
    bgs_context* ctx;            // NULL once the context is destroyed
    std::vector<ListEntity> ent;
    uint64_t total = 0;          // N
    std::map<const bgs_cloud*, uint32_t> clouds;   // entities per listed cloud (detached ones not counted)
    std::map<uint32_t, std::array<uint32_t, 2>> groups;   // entities per projection group, and of those reading SH
    uint32_t kinds[3] = {0, 0, 0};   // entities per blend kind
    uint32_t boxed = 0, depth = 0, flow = 0, detached = 0;   // entities with the overlay bit, in Depth, in OpticalFlow, detached
    // non-4D Velocity entities per (gaussian_mode, aabb, opacity_adaptive_radius, draw_mode, overlay bit): [0] with the
    // entity's own overlay bit, [1] with the bit set (frames with the frame-wide overlay)
    std::map<std::array<uint32_t, 5>, uint32_t> velocity[2];
    std::shared_ptr<ListTable> cur, spare;   // the generation edits and frames use; one a frame held, for reuse
    DevBuf<uint8_t> upload;      // the edits' records on their way to the scatter
};

namespace bgs {

// live contexts: clouds may be shared by the contexts of one GPU, so destroying a cloud must clear every context's
// references to it, and a write to a cloud must wait for every context's frames that may read it
extern std::mutex g_registry_mu;
extern std::vector<bgs_context*> g_contexts;
// live entity lists (bgs_entity_list): destroying a cloud detaches the entities that list it (api.cu), under the registry lock
extern std::vector<bgs_entity_list*> g_lists;
void detach_listed_cloud(const bgs_cloud* cl);

// Sets the context's last-error text (when there is a context) and returns `st`.
bgs_status fail(bgs_context* ctx, bgs_status st, const char* fmt, ...);

inline bgs_status status_of(cudaError_t e) { return e == cudaErrorMemoryAllocation ? BGS_ENOMEM : BGS_ECUDA; }

#define CU(ctx, call)                                                                                  \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) return fail(ctx, status_of(e_), "%s: %s", #call, cudaGetErrorString(e_)); \
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
        return fail(c, status_of(e), "allocating %zu bytes of device scratch: %s", want, cudaGetErrorString(e));
    }
    p = static_cast<T*>(np);
    bytes = want;
    return BGS_OK;
}

// The preamble of every call on a resident cloud or behaviours object, after its null-argument checks: a context, the
// object on the context's device (`what` names it in the message), and that device current.
inline bgs_status enter_call(bgs_context* c, const char* call, int device, const char* what = "cloud lives") {
    if (!c) return BGS_EINVAL;
    if (device != c->device) return fail(c, BGS_EINVAL, "%s: %s on another device", call, what);
    CU(c, cudaSetDevice(c->device));
    return BGS_OK;
}

// ---- The order of a cloud's accesses (clouds are shared by the contexts of one GPU), on the context's render stream.
// Read: after every particle step queued on the cloud, on the device (one wait, and only once it has been stepped).
// Synchronous write: the same, once the host has completed every frame queued on the cloud's GPU, this context's through
// bgs_sync (whose failure is returned).  Queued write (the step): on the device, after every frame queued on any
// context of the GPU (each context's ev_done marks its last) and every earlier step of the cloud, under the registry
// lock so another context's write waits and records in turn; it then marks itself on the cloud's ev_write.
// Queued write that reads other clouds (the interpolation): the queued write's order, after the read order of each
// input; it then re-records the context's ev_done and sets reads_pending, so that a later queued write of an input waits
// for it on the device and a later synchronous write or destroy of an input drains it on the host.

inline bgs_status before_cloud_read(bgs_context* c, const bgs_cloud* cl) {
    if (cl->stepped.load(std::memory_order_acquire)) CU(c, cudaStreamWaitEvent(c->stream, cl->ev_write, 0));
    return BGS_OK;
}

inline bgs_status before_cloud_write(bgs_context* c, const bgs_cloud* cl) {
    if (c->async_pending) TRY(bgs_sync(c));
    TRY(before_cloud_read(c, cl));
    std::lock_guard<std::mutex> lk(g_registry_mu);
    for (bgs_context* o : g_contexts)
        if (o != c && o->device == cl->device && (o->async_pending || o->reads_pending.load(std::memory_order_relaxed)))
            o->each_stream([](cudaStream_t& s, int) { cudaStreamSynchronize(s); });
    return BGS_OK;
}

// `write(stream)` enqueues the write itself
template <class Write>
bgs_status queue_cloud_write(bgs_context* c, bgs_cloud* cl, Write write) {
    cudaStream_t q = c->stream;
    std::lock_guard<std::mutex> lk(g_registry_mu);
    if (!cl->ev_write) CU(c, cudaEventCreateWithFlags(&cl->ev_write, cudaEventDisableTiming));
    for (bgs_context* o : g_contexts)
        if (o != c && o->device == c->device) CU(c, cudaStreamWaitEvent(q, o->ev_done, 0));
    if (cl->stepped.load(std::memory_order_relaxed)) CU(c, cudaStreamWaitEvent(q, cl->ev_write, 0));
    TRY(write(q));
    CU(c, cudaEventRecord(cl->ev_write, q));
    cl->stepped.store(true, std::memory_order_release);
    return BGS_OK;
}

// `write(stream)` enqueues the write of `cl`, which reads `in0` and `in1`
template <class Write>
bgs_status queue_cloud_write_reading(bgs_context* c, bgs_cloud* cl, const bgs_cloud* in0, const bgs_cloud* in1, Write write) {
    return queue_cloud_write(c, cl, [&](cudaStream_t q) {
        TRY(before_cloud_read(c, in0));
        if (in1 != in0) TRY(before_cloud_read(c, in1));
        TRY(write(q));
        CU(c, cudaEventRecord(c->ev_done, q));
        c->reads_pending.store(true, std::memory_order_relaxed);
        return BGS_OK;
    });
}

// the frame constants the render calls build for a cloud, uniform, view and settings (api.cu); bgs_cloud_select_in_view
// builds its own with them
FrameConsts frame_consts(const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uni, const bgs_settings* st,
                         bool want_aux);

// ---- frame scratch (api.cu) that the selections borrow
int pair_passes(uint32_t num_tiles);
bgs_status ensure_cloud_scratch(bgs_context* c, uint32_t n);
bgs_status ensure_status(bgs_context* c, DevBuf<void>& rows, uint32_t& rows_capacity, uint32_t capacity);
uint32_t next_epoch(bgs_context* c);

}  // namespace bgs
