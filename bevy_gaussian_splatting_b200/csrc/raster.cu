// raster.cu -- stage 5: per-16x16-tile front-to-back alpha blend.
//
// Replaces the reference's instanced-quad draw + fixed-function ROP blending
// (vs_points/fs_main, src/render/gaussian.wgsl:185-505; PREMULTIPLIED_ALPHA_BLENDING applied
// far->near, src/render/mod.rs:944-948).  Per pixel, the same coverage rule (pixel centre inside
// the splat's OBB quad, |u|<=1 and |v|<=1), the same falloff (alpha = min(exp(-4.5|uv|^2) * o *
// g_o, 0.999), gaussian.wgsl:474-504) and the same "over" operator, evaluated front-to-back:
//   C = sum_j rgb_j a_j T_j,  T_j = prod_{k nearer}(1 - a_k);   out = C + T*background(=0), a=1.
// A pixel stops once T < 1e-4; a tile stops when all its pixels have stopped (block vote).
//
// One CTA per tile, 256 threads = 8 warps, each warp owning an 8x4-pixel sub-rectangle so a
// warp-uniform bbox test skips splats that cannot touch any of its 32 pixels.  The tile's slice
// of the sorted pair list is staged through shared memory in chunks of 256 records.
// Coverage maths (quad_uv) uses explicit __fmul_rn/__fmaf_rn so u,v are bit-identical to the oracle.
#include <cuda_fp16.h>

#include <type_traits>
#include <utility>

#include "common.cuh"
#include "launch.cuh"
#include "pixel.cuh"

namespace bgs {

constexpr int RT_THREADS = 256;
constexpr int RT_CHUNK = 256;

// ---- TMA (cp.async.bulk) staging of a tile's slice of the sorted pair list ------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
constexpr uint32_t ENT_WORDS = RT_CHUNK + 8;   // a chunk plus up to 3 leading + rounding words

// A tile's slice [range.x, range.y) of tile_entries, chunk by chunk: per chunk (loop index `chunk`, first entry `base`)
// next(base), then entry(base, j); finish() after the loop.  A streamed slice (`tma`, the kernel's choice) comes into the
// double buffer `ent` by ONE bulk async copy (UBLKCP) per chunk, issued by thread 0 and tracked by an mbarrier; chunk
// k + 1's copy is in flight while chunk k is blended.  Bulk copies need 16 B alignment: a copy starts at the slice
// address rounded down to 16 B and entry() skips the `base & 3` leading words.  Other slices are read from global memory.
struct PairStream {
    const uint32_t* entries;
    uint32_t (*ent)[ENT_WORDS];
    uint32_t a_ent, a_bar, end;
    bool tma;
    uint32_t issued = 0u, chunk = 0u;   // bulk copies issued; chunks [0, chunk) have been waited for

    // collective when `tma`: initialises the barriers, then issues chunk 0's copy
    __device__ __forceinline__ PairStream(const uint32_t* tile_entries, uint32_t (*s_ent)[ENT_WORDS], unsigned long long* s_bar,
                                          uint2 range, bool use_tma)
        : entries(tile_entries), ent(s_ent), a_ent((uint32_t)__cvta_generic_to_shared(s_ent)),
          a_bar((uint32_t)__cvta_generic_to_shared(s_bar)), end(range.y), tma(use_tma) {
        if (!tma) return;
        if (threadIdx.x == 0) {
            mbar_init(a_bar, 1u); mbar_init(a_bar + 8u, 1u);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) issue(range.x, (uint32_t)RT_CHUNK, 0);
        issued = 1u;
    }
    // bulk copy of entries [base, base + cnt) into buffer `buf` (thread 0 only)
    __device__ __forceinline__ void issue(uint32_t base, uint32_t cnt, int buf) const {
        const uint32_t lead = base & 3u;
        const uint32_t bytes = ((lead + cnt) * 4u + 15u) & ~15u;
        mbar_expect_tx(a_bar + 8u * buf, bytes);
        tma_bulk_g2s(a_ent + (uint32_t)buf * ENT_WORDS * 4u, entries + (base - lead), bytes, a_bar + 8u * buf);
    }
    // chunk `chunk` starts at `base`: prefetch the NEXT chunk's entries (its buffer was last read two chunks ago, which
    // the kernel's vote at the top of this chunk fenced), then wait for this one's
    __device__ __forceinline__ void next(uint32_t base) {
        const int buf = (int)(chunk & 1u);
        if (tma) {
            if (base + RT_CHUNK < end) {
                if (threadIdx.x == 0) issue(base + RT_CHUNK, min((uint32_t)RT_CHUNK, end - base - RT_CHUNK), buf ^ 1);
                ++issued;
            }
            mbar_wait(a_bar + 8u * buf, (chunk >> 1) & 1u);
        }
    }
    template <class Index>   // int or uint32_t, as the caller's loop has it
    __device__ __forceinline__ uint32_t entry(uint32_t base, Index j) const {
        return tma ? ent[chunk & 1u][(base & 3u) + j] : __ldg(entries + base + j);
    }
    // an early exit (all pixels saturated) may leave one prefetch in flight: keep the CTA alive until it lands
    __device__ __forceinline__ void finish() const {
        if (threadIdx.x == 0 && issued > chunk) mbar_wait(a_bar + 8u * (chunk & 1u), (chunk >> 1) & 1u);
    }
};

// CTA -> tile: rows are visited from the middle row outwards (mid, mid-1, mid+1, ...), so the tiles launched last --
// the ones that form the kernel's tail -- are the top / bottom rows, usually the lightest.
__device__ __forceinline__ void centre_out_tile(int b, int tiles_x, int tiles_y, int& tile_x, int& tile_y) {
    const int k = b / tiles_x, mid = tiles_y / 2;
    tile_x = b - k * tiles_x;
    tile_y = (k & 1) ? mid - (k + 1) / 2 : mid + k / 2;
}

// shared-memory layout (byte offsets from one base so the hot loop needs a single address register)
constexpr uint32_t SM_Q0 = 0;                         // float4 [256]: cx, cy, ux, uy
constexpr uint32_t SM_UV = SM_Q0 + RT_CHUNK * 16;     // float4 [256]: vx, vy, bbox x, bbox y
constexpr uint32_t SM_Q2 = SM_UV + RT_CHUNK * 16;     // float4 [256]: r, g, b, opacity
constexpr uint32_t SM_LIST = SM_Q2 + RT_CHUNK * 16;   // u16 [8][256]: per-warp candidates, stored as index * 16
constexpr uint32_t SM_EXTRA = SM_LIST + (RT_THREADS / 32) * RT_CHUNK * 2;   // MODE 2 only: 4 x float4 [256]
constexpr uint32_t SM_BYTES = SM_EXTRA;
constexpr uint32_t SM_BYTES_2D = SM_EXTRA + 4 * RT_CHUNK * 16;
// AUX (bgs_render_aux): 2 x float4 [256] after the mode's own arrays: depth rgb, normal rgb of the staged splats
// ZTEST (bgs_render_depth_test): float [256] at a 16 B stride after the mode's own arrays: the staged splats' depths d,
// at the same offset from a splat's q0 record for every splat (what the candidate lists hold), so the blend loops reach
// d with one load from the record address.  AUX + ZTEST (bgs_render_entities_aux with a depth buffer): d rides in the
// unused w lane of the staged depth colour instead, so MODE 4's arrays (40 KB) and the CTA's other shared arrays stay
// within the 48 KB static limit
constexpr uint32_t ZT_BYTES = RT_CHUNK * 16;

// a staged splat's uv and q2 records, as offsets from the shared address of its q0 record (what the candidate lists hold)
constexpr uint32_t REC_UV = SM_UV - SM_Q0, REC_Q2 = SM_Q2 - SM_Q0;
static_assert(REC_UV == RT_CHUNK * 16 && REC_Q2 == 2 * RT_CHUNK * 16, "q0, uv, q2 are consecutive float4 [RT_CHUNK] arrays");

// loads from a shared address (volatile: they keep their order in the hot loops)
__device__ __forceinline__ float4 lds4(uint32_t a) {
    float4 r; asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(a)); return r;
}
__device__ __forceinline__ float2 lds2(uint32_t a) {
    float2 r; asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "r"(a)); return r;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) { uint32_t r; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(r) : "r"(a)); return r; }

// USE_OBB quad coordinates of the pixel centre (fx, fy) for q0 = (cx, cy, ux, uy), q1 = (vx, vy): u = ux dx + uy dy with
// the fma on the dy term, v likewise.  The same rounding steps as decide() in oracle/bgs_oracle.cpp, so the coverage
// test |u|, |v| <= 1 is bit-identical to the oracle's.
__device__ __forceinline__ float2 quad_uv(float fx, float fy, float4 q0, float2 q1) {
    const float dx = __fsub_rn(fx, q0.x), dy = __fsub_rn(fy, q0.y);
    return make_float2(__fmaf_rn(q0.w, dy, __fmul_rn(q0.z, dx)), __fmaf_rn(q1.y, dy, __fmul_rn(q1.x, dx)));
}

// bgs_render_depth_test: the scene depth of pixel (px, py), row pitch in bytes; pixels outside the frame are never read
// and get NaN, which the warp's minimum ignores and which blends nothing (those pixels are stopped from the start)
__device__ __forceinline__ float scene_depth_at(const float* scene, size_t pitch, int px, int py, bool inside) {
    return inside ? __ldg(reinterpret_cast<const float*>(reinterpret_cast<const char*>(scene) + (size_t)py * pitch) + px)
                  : __uint_as_float(0x7FC00000u);
}
// the minimum over the warp's pixels, NaN ignored (fminf): a splat whose d is below it fails d >= scene at every pixel of
// the warp's rectangle, so the candidate compaction may drop it without changing any decision
__device__ __forceinline__ float warp_min_depth(float z) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z = fminf(z, __shfl_xor_sync(0xffffffffu, z, o));
    return z;
}
__device__ __forceinline__ float lds_f32(uint32_t a) { float r; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r) : "r"(a)); return r; }

// BOX (BGS_FLAG_VISUALIZE_BOUNDING_BOX, gaussian.wgsl:486-495): the pair lies on its quad's edge band when s = uv / 2 + 1/2
// is within 0.08 of 0 or 1 on either axis (a NaN component is not an edge).  uv is the quad uv of a quad-uv splat and
// m / R of a conic or surfel one.
constexpr float BOX_EDGE = 0.08f;
__device__ __forceinline__ bool box_edge(float u, float v) {
    const float sx = __fadd_rn(__fmul_rn(u, 0.5f), 0.5f), sy = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);
    return sx < BOX_EDGE || sx > 1.0f - BOX_EDGE || sy < BOX_EDGE || sy > 1.0f - BOX_EDGE;
}

// Each warp compacts the chunk's `cnt` staged splats to those `hit(j)` keeps, in order, into its u16 list as
// `rec0 + j * 16` (the q0 record's address relative to rec0); returns the list's length.
template <class Hit>
__device__ __forceinline__ uint32_t compact_candidates(uint32_t cnt, unsigned short* list, uint32_t rec0, Hit hit) {
    uint32_t nl = 0;
    for (uint32_t j0 = 0; j0 < cnt; j0 += 32) {
        const uint32_t j = j0 + (threadIdx.x & 31u);
        bool h = false;
        if (j < cnt) h = hit(j);
        const uint32_t m = __ballot_sync(0xffffffffu, h);
        if (h) list[nl + __popc(m & lanemask_lt())] = (unsigned short)(rec0 + j * 16u);
        nl += __popc(m);
    }
    __syncwarp();
    return nl;
}

// MODE 0: USE_OBB quad-uv falloff (3DGS, and 2DGS without aabb)   gaussian.wgsl:474-504
// MODE 1: 3DGS USE_AABB conic falloff                              gaussian.wgsl:459-471
// MODE 2: 2DGS USE_AABB ray-splat intersection                     gaussian.wgsl:441-458, gaussian_2d.wgsl:134-156
// AUX: the same pass also blends the splats' Depth and Normal colour sources (aux records, 2 x float4 per splat) into two
// more frames with the very same alphas: config C4's colour + depth + normal outputs cost one pass, not three.  Every
// mode takes it (bgs_render_aux: MODE 0, 1, 2; bgs_render_entities_aux: any MODE, with or without ZTEST and BOX).
// ZTEST: bgs_render_depth_test.  A pair blends only where its coverage decision holds and
// d >= the pixel's scene depth; the warp's candidates leave out the splats below the scene everywhere in its rectangle.
// MODE 3 / 4 (bgs_render_entities): mixed kinds, each splat tested by its own: kinds[r] (raster_kinds_kernel) is record r's
// 0 = quad-uv, 1 = conic, 2 = surfel; MODE 4 when some splat is a surfel (the only one that stages the surfel records).
// Warp candidates: bbox for every kind, and the separating-axis test of MODE 0 for the quad-uv splats.
// BOX (BGS_FLAG_VISUALIZE_BOUNDING_BOX): the bounding-box overlay.  A covered pair (after the aabb discard and the depth
// test) on its quad's edge band (box_edge) blends (0.3, 1, 0.1) at alpha 1 into every frame it writes, which stops the
// pixel; other pairs blend as without it.  Mixed frames read the overlay bit of each splat from bit 2 of its kinds byte
// (its entity's), the others draw every splat's box.  MODE 0 takes the generic loop, not the inline-asm one.
// VIEWS (raster_kernel's ViewTable variants, bgs_render_views): the CTA's global tile blockIdx.x lies in view
// i = vt->view_of_tile; W, H, tiles_x, out, scene and pitch are then view i's, the CTA takes the local tile
// blockIdx.x - tile0[i] in centre_out_tile's order within the view, and reads the global tile's range.  With AUX
// (bgs_render_views_aux) out_depth and out_normal are view i's too.
// PICK (raster_kernel's PickArgs variants, bgs_render_entities_pick): beside its colour each pixel keeps the largest
// weight w = a T of the pairs it blends (an overlay edge pair: w = T) and that pair's record; a later pair replaces it only
// when its w is strictly larger.  Every pixel of pk->out is written: (entity, index, w, d) of that pair, or BGS_PICK_NONE
// where nothing blends.  Pick frames take the generic loop in every mode, never the inline-asm one.
// RAW (raster_kernel's SubFrames variants, bgs_render_shutter; with VIEWS): each pixel stores its raw blended state
// (C, T) as a float4 into its view's out, before any output mode, and an empty tile stores (0, 0, 0, 1); format is not
// read.  The resolve (shutter.cu) encodes the frame from those states.
template <int MODE, bool AUX, bool ZTEST, bool BOX = false, bool VIEWS = false, bool PICK = false, class Pick = PickArgs,
          bool RAW = false>
__device__ __forceinline__ void raster_body(const SplatRec* __restrict__ recs, const float4* __restrict__ extra,
                                            const uint32_t* __restrict__ tile_entries, const uint2* __restrict__ ranges, int W,
                                            int H, int tiles_x, void* __restrict__ out, uint32_t format,
                                            const float4* __restrict__ aux, void* __restrict__ out_depth,
                                            void* __restrict__ out_normal, const uint32_t* __restrict__ truncated,
                                            const float* __restrict__ splat_d, const float* __restrict__ scene, size_t pitch,
                                            const unsigned char* __restrict__ kinds, const ViewTable* vt = nullptr,
                                            const Pick* pk = nullptr) {
    constexpr bool MIXED = MODE >= 3, SURF = MODE == 2 || MODE == 4;
    __shared__ __align__(16) unsigned char s_mem[(SURF ? SM_BYTES_2D : SM_BYTES) + (AUX ? 2 * RT_CHUNK * 16 : 0) +
                                                 (ZTEST && !AUX ? ZT_BYTES : 0)];
    constexpr uint32_t SM_AUX = SURF ? SM_BYTES_2D : SM_BYTES;
    // ZTEST: d of the splat whose q0 record is at a, at a + REC_D (AUX: the w lane of its staged depth colour)
    constexpr uint32_t REC_D = AUX ? SM_AUX + 12 : SM_AUX;
    __shared__ __align__(16) uint32_t s_ent[2][ENT_WORDS];    // TMA destination: the tile's pair-list chunks
    __shared__ __align__(8) unsigned long long s_bar[2];
    // MODE 0 and mixed: per staged splat cull thresholds (u, v) (quad-uv splats only)
    __shared__ __align__(8) float2 s_thr[MODE == 0 || MIXED ? RT_CHUNK : 1];
    __shared__ unsigned char s_kind[MIXED ? RT_CHUNK : 1];   // mixed: the staged splats' kinds
    float4* s_q0 = reinterpret_cast<float4*>(s_mem + SM_Q0);
    float4* s_uv = reinterpret_cast<float4*>(s_mem + SM_UV);
    float4* s_q2 = reinterpret_cast<float4*>(s_mem + SM_Q2);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    unsigned short* s_list = reinterpret_cast<unsigned short*>(s_mem + SM_LIST) + warp * RT_CHUNK;
    const uint32_t a_base = (uint32_t)__cvta_generic_to_shared(s_mem);
    const uint32_t a_list = a_base + SM_LIST + (uint32_t)warp * RT_CHUNK * 2u;
    int tile_x, tile_y, tile;
    if constexpr (VIEWS) {
        const uint32_t i = vt->view_of_tile(blockIdx.x);
        W = vt->W[i]; H = vt->H[i]; tiles_x = vt->tiles_x[i]; out = vt->out[i];
        if (ZTEST) { scene = vt->scene[i]; pitch = vt->pitch[i]; }
        if (AUX) { out_depth = vt->out_depth[i]; out_normal = vt->out_normal[i]; }
        centre_out_tile((int)(blockIdx.x - vt->tile0[i]), tiles_x, vt->tiles_y[i], tile_x, tile_y);
        tile = (int)vt->tile0[i] + tile_y * tiles_x + tile_x;
    } else {
        centre_out_tile((int)blockIdx.x, tiles_x, (int)gridDim.x / tiles_x, tile_x, tile_y);
        tile = tile_y * tiles_x + tile_x;
    }
    // warp w covers the 8x4 rectangle at ((w & 1) * 8, (w >> 1) * 4) of the tile
    const int wx0 = tile_x * TILE_PX + (warp & 1) * 8, wy0 = tile_y * TILE_PX + (warp >> 1) * 4;
    const int px = wx0 + (lane & 7), py = wy0 + (lane >> 3);
    const bool inside = px < W && py < H;
    const float fx = (float)px + 0.5f, fy = (float)py + 0.5f;
    const float rcx = (float)wx0 + 4.0f, rcy = (float)wy0 + 2.0f;   // centre of the warp's pixel centres
    const float tcx = (float)(tile_x * TILE_PX) + 8.0f, tcy = (float)(tile_y * TILE_PX) + 8.0f;   // tile centre
    uint2 range = ranges[tile];
    // a pair list cut short by the buffer's capacity: the frame is rendered again after the buffer grows, so this attempt
    // leaves every target as it was (blend-over must not composite the layer twice).  (Loaded beside the range, and not
    // kept live through the blend: the register budget of raster_kernel<0> has no room for it.)
    if (*truncated) return;
    range.x = ~range.x;                  // stored as (~start, end): the sort's last pass builds it with atomicMax (radix.cu)

    if (range.x >= range.y) {            // empty tile: nothing to stage (uniform across the CTA)
        // (blend-over mode leaves the target's pixels as they are)
        if (PICK && inside) pk->out[(size_t)py * W + px] = make_uint4(BGS_PICK_NONE, BGS_PICK_NONE, 0u, 0u);
        if (RAW && inside) reinterpret_cast<float4*>(out)[(size_t)py * W + px] = make_float4(0.f, 0.f, 0.f, 1.0f);
        if (!RAW && inside && !((format >> 8) & OUT_OVER)) {
            write_pixel(out, format, (size_t)py * W + px, 0.f, 0.f, 0.f, 1.0f);
            if (AUX) {
                write_pixel(out_depth, format, (size_t)py * W + px, 0.f, 0.f, 0.f, 1.0f);
                write_pixel(out_normal, format, (size_t)py * W + px, 0.f, 0.f, 0.f, 1.0f);
            }
        }
        return;
    }
    // tiles with more than one chunk stream their pair list (the next chunk's copy overlaps this chunk's blending)
    PairStream ps(tile_entries, s_ent, s_bar, range, range.y - range.x > (uint32_t)RT_CHUNK);
    float zs = 0.0f, zmin = 0.0f;   // ZTEST: this pixel's scene depth, the minimum over the warp's pixels
    if (ZTEST) {
        zs = scene_depth_at(scene, pitch, px, py, inside);
        zmin = warp_min_depth(zs);
    }

    float T = inside ? 1.0f : 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;   // T < T_STOP <=> this pixel is done
    float dr = 0.0f, dg = 0.0f, db = 0.0f, nr = 0.0f, ng = 0.0f, nb = 0.0f;   // AUX: depth / normal frames
    float best_w = -1.0f;               // PICK: the largest w so far (-1: none), and its record
    uint32_t best_r = BGS_PICK_NONE;
    for (uint32_t base = range.x; base < range.y; base += RT_CHUNK, ++ps.chunk) {
        if (__syncthreads_count(T < T_STOP ? 0 : 1) == 0) break;   // also fences reuse of the staging buffers
        const uint32_t cnt = min((uint32_t)RT_CHUNK, range.y - base);
        ps.next(base);
        if ((uint32_t)t < cnt) {
            const uint32_t r = ps.entry(base, t);
            const float4* rp = reinterpret_cast<const float4*>(recs + r);
            const float4 p0 = __ldg(rp), p1 = __ldg(rp + 1);
            s_q0[t] = p0;
            s_uv[t] = p1;
            s_q2[t] = __ldg(rp + 2);
            const int kb = MIXED ? (int)__ldg(kinds + r) : MODE;   // BOX: kind | overlay << 2
            if (MIXED) s_kind[t] = (unsigned char)kb;
            const int kind = BOX ? (kb & 3) : kb;
            if (kind == 0) {
                // thresholds of the per-warp separating-axis cull below, once per splat: the quad |u| <= 1, |v| <= 1
                // misses a warp rectangle (pixel centres within +-3.5 x +-1.5 of its centre) when |u(centre)| exceeds
                // 1 + |ux| 3.5 + |uy| 1.5 (same for v).  Slack: 1e-5 of the largest magnitude the terms of u can take
                // anywhere in the tile, ~100x the rounding error of the per-pixel u, v.  NaN/inf never cull.
                const float ax = fabsf(p0.x - tcx) + 4.0f, ay = fabsf(p0.y - tcy) + 6.0f;
                const float ur = fabsf(p0.z) * 3.5f + fabsf(p0.w) * 1.5f, vr = fabsf(p1.x) * 3.5f + fabsf(p1.y) * 1.5f;
                const float um = fabsf(p0.z) * ax + fabsf(p0.w) * ay + ur, vm = fabsf(p1.x) * ax + fabsf(p1.y) * ay + vr;
                s_thr[t] = make_float2(ur + 1.0f + 1e-5f * um, vr + 1.0f + 1e-5f * vm);
            }
            if (SURF && kind == 2) {
                float4* s_ex = reinterpret_cast<float4*>(s_mem + SM_EXTRA);
                const float4* ep = extra + (size_t)r * 4;
#pragma unroll
                for (int q = 0; q < 4; ++q) s_ex[q * RT_CHUNK + t] = __ldg(ep + q);
            }
            if (AUX) {
                float4* s_ax = reinterpret_cast<float4*>(s_mem + SM_AUX);
                float4 ad = __ldg(aux + (size_t)r * 2);
                if (ZTEST) ad.w = __ldg(splat_d + r);   // (REC_D; the blend reads the colour's x, y, z only)
                s_ax[t] = ad;
                s_ax[RT_CHUNK + t] = __ldg(aux + (size_t)r * 2 + 1);
            }
            if (ZTEST && !AUX) reinterpret_cast<float*>(s_mem + REC_D)[4 * t] = __ldg(splat_d + r);
        }
        __syncthreads();
        // each warp's candidates: the splats whose bbox touches its 8x4 pixels, listed by shared address of q0[j]
        const uint32_t nl = !__any_sync(0xffffffffu, !(T < T_STOP)) ? 0u : compact_candidates(cnt, s_list, a_base, [&](uint32_t j) {
            const float4 q = s_uv[j];
            const uint32_t bx = __float_as_uint(q.z), by = __float_as_uint(q.w);
            // (`|`, not `||`: the four compares are one predicated test, not a chain of branches)
            bool hit = !((int)(bx >> 16) < wx0 | (int)(bx & 0xFFFFu) > wx0 + 7 | (int)(by >> 16) < wy0 |
                         (int)(by & 0xFFFFu) > wy0 + 3);
            if ((MODE == 0 || (MIXED && (BOX ? (s_kind[j] & 3) : s_kind[j]) == 0)) && hit) {
                // separating-axis test of the splat's quad against this warp's pixel centres
                // [wx0 + .5, wx0 + 7.5] x [wy0 + .5, wy0 + 3.5] (thresholds staged per splat above): the bbox
                // of a slanted quad passes many warps none of whose pixels it covers
                const float4 p = s_q0[j];
                const float2 th = s_thr[j];
                const float dxc = rcx - p.x, dyc = rcy - p.y;
                hit = !(fabsf(p.z * dxc + p.w * dyc) > th.x || fabsf(q.x * dxc + q.y * dyc) > th.y);
            }
            if (ZTEST && hit) hit = !(reinterpret_cast<const float*>(s_mem + REC_D)[4 * j] < zmin);
            return hit;
        });
        if (MODE == 0 && !AUX && !BOX && !PICK) {
            // four candidates per iteration, so loop control is paid once per four; each list entry is its own 16-bit
            // load (cheaper than unpacking a 32-bit pair); blending stays strictly in list order.
            // The blend is PREDICATED, not branched: 15 SASS instructions per candidate instead of a divergent block
            // with its BSSY / BRA / BREAK / BSYNC bookkeeping (~23 issue slots; 98 % of the candidates cover some pixel of
            // the warp anyway).  A candidate blends where it covers the pixel and T >= T_STOP: a stopped pixel (and one
            // outside the frame, T = 0) skips every later splat exactly as an early exit would, and the stop costs one
            // `setp ... .and` of the T the previous blend left, instead of a stop flag updated after every blend.
            const uint32_t a_end = a_list + nl * 2u, a_end4 = a_end - 6u;   // (no wrap: a_list >= SM_LIST)
            uint32_t a_it = a_list;
            // ZTEST: one more load and one more `setp ... .and`: the pair blends only where d >= the scene depth (%8)
#define BLEND_COVER_                                                                                                    \
                    "{\n\t"                                                                                             \
                    ".reg .pred p;\n\t"                                                                                 \
                    ".reg .f32 au, av, x, y, z, o, qd, e, a, w, na;\n\t"                                                \
                    "abs.f32 au, %4;\n\t"                                                                               \
                    "abs.f32 av, %5;\n\t"                                                                               \
                    "setp.le.f32 p, au, 0f3F800000;\n\t"                                                                \
                    "setp.le.and.f32 p, av, 0f3F800000, p;\n\t"                                                         \
                    "setp.ge.and.f32 p, %0, 0f38D1B717, p;\n\t"   /* alive: T >= T_STOP (1e-4f) */
#define BLEND_ZTEST_                                                                                                    \
                    ".reg .f32 dz;\n\t"                                                                                \
                    "ld.shared.f32 dz, [%6+%9];\n\t"                                                                    \
                    "setp.ge.and.f32 p, dz, %8, p;\n\t"
                    // (the temporaries are computed unconditionally -- a predicated definition would keep their old values
                    // alive across iterations -- only the four accumulations are predicated)
#define BLEND_ACCUMULATE_                                                                                               \
                    "ld.shared.v4.f32 {x, y, z, o}, [%6+%7];\n\t"                                                       \
                    "mul.rn.f32 qd, %4, %4;\n\t"                                                                        \
                    "fma.rn.f32 qd, %5, %5, qd;\n\t"                                                                    \
                    "mul.rn.f32 qd, qd, 0fC0CFBF83;\n\t"     /* -6.492127684f: exp(-4.5 qd) = 2^(qd * -4.5 log2 e) */  \
                    "ex2.approx.ftz.f32 e, qd;\n\t"                                                                     \
                    "mul.rn.f32 a, e, o;\n\t"                                                                           \
                    "min.f32 a, a, 0f3F7FBE77;\n\t"          /* 0.999f */                                               \
                    "mul.rn.f32 w, a, %0;\n\t"                                                                          \
                    "neg.f32 na, a;\n\t"                                                                                \
                    "@p fma.rn.f32 %1, w, x, %1;\n\t"                                                                   \
                    "@p fma.rn.f32 %2, w, y, %2;\n\t"                                                                   \
                    "@p fma.rn.f32 %3, w, z, %3;\n\t"                                                                   \
                    "@p fma.rn.f32 %0, na, %0, %0;\n\t"                                                                 \
                    "}"
            auto blend_if_covered = [&](uint32_t a_rec, float2 uv) {
                if constexpr (ZTEST)
                    asm volatile(BLEND_COVER_ BLEND_ZTEST_ BLEND_ACCUMULATE_
                                 : "+f"(T), "+f"(cr), "+f"(cg), "+f"(cb)
                                 : "f"(uv.x), "f"(uv.y), "r"(a_rec), "n"(REC_Q2), "f"(zs), "n"(REC_D));
                else
                    asm volatile(BLEND_COVER_ BLEND_ACCUMULATE_
                                 : "+f"(T), "+f"(cr), "+f"(cg), "+f"(cb)
                                 : "f"(uv.x), "f"(uv.y), "r"(a_rec), "n"(REC_Q2));
            };
#undef BLEND_COVER_
#undef BLEND_ZTEST_
#undef BLEND_ACCUMULATE_
            for (; a_it < a_end4; a_it += 8u) {
                const uint32_t ra = lds_u16(a_it), rb = lds_u16(a_it + 2u), rc = lds_u16(a_it + 4u), rd = lds_u16(a_it + 6u);
                blend_if_covered(ra, quad_uv(fx, fy, lds4(ra), lds2(ra + REC_UV)));
                blend_if_covered(rb, quad_uv(fx, fy, lds4(rb), lds2(rb + REC_UV)));
                blend_if_covered(rc, quad_uv(fx, fy, lds4(rc), lds2(rc + REC_UV)));
                blend_if_covered(rd, quad_uv(fx, fy, lds4(rd), lds2(rd + REC_UV)));
            }
#pragma unroll 1
            for (; a_it != a_end; a_it += 2u) {   // the last nl % 4
                const uint32_t ra = lds_u16(a_it);
                blend_if_covered(ra, quad_uv(fx, fy, lds4(ra), lds2(ra + REC_UV)));
            }
        } else if (!(T < T_STOP)) {
            const uint32_t a_end = a_list + nl * 2u;
            for (uint32_t a_it = a_list; a_it != a_end; a_it += 2u) {
                const uint32_t a_rec = lds_u16(a_it);
                const float4 q0 = lds4(a_rec);
                const float2 q1 = lds2(a_rec + REC_UV);
                // ZTEST: the depth test joins each mode's coverage test (d >= scene; a NaN on either side fails)
                auto depth_ok = [&]() { return !ZTEST || lds_f32(a_rec + REC_D) >= zs; };
                float e;
                float4 q2;
                const int kb = MIXED ? (int)s_kind[(a_rec - a_base) >> 4] : MODE;
                const int kind = BOX ? (kb & 3) : kb;
                const bool box = BOX && (!MIXED || (kb >> 2) != 0);   // this splat's overlay
                bool edge = false;                                     // BOX: the pair is on its quad's edge band
                if (kind == 0) {
                    const float2 uv = quad_uv(fx, fy, q0, q1);
                    if (!(fabsf(uv.x) <= 1.0f && fabsf(uv.y) <= 1.0f && depth_ok())) continue;
                    if (BOX) edge = box && box_edge(uv.x, uv.y);
                    const float qd = __fmaf_rn(uv.y, uv.y, __fmul_rn(uv.x, uv.x));
                    q2 = lds4(a_rec + REC_Q2);
                    // exp(-4.5 qd) = 2^(qd * -4.5 log2 e); qd <= 2 so the argument stays >= -13 (no range fix-up)
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(qd * -6.492127684f));
                } else {
                    // quad-space offset in half-pixels (x right, y up); the quad is the square |m| <= Rq
                    const float dx = __fsub_rn(fx, q0.x), dy = __fsub_rn(fy, q0.y);
                    const float mx = __fadd_rn(dx, dx), my = -__fadd_rn(dy, dy);
                    const float Rq = q1.y;   // MODE 1: quad half-side in half-pixels
                    float power, R = Rq;     // R: the half-side the coverage test compares |m| against
                    if (kind == 1 || !SURF) {
                        if (!(fabsf(mx) <= Rq && fabsf(my) <= Rq && depth_ok())) continue;
                        // q0.z, q0.w, q1.x = conic x, y, z;  d = -m  (gaussian.wgsl:459-462)
                        const float ddx = -mx, ddy = -my;
                        const float t1 = __fmul_rn(__fmul_rn(q0.z, ddx), ddx), t2 = __fmul_rn(__fmul_rn(q1.x, ddy), ddy);
                        power = __fadd_rn(__fmul_rn(-0.5f, __fadd_rn(t1, t2)), __fmul_rn(__fmul_rn(q0.w, ddx), ddy));
                    } else {
                        const float4 e0 = lds4(a_rec + SM_EXTRA);
                        if (!(fabsf(mx) <= e0.x && fabsf(my) <= e0.x && depth_ok())) continue;
                        if (BOX) R = e0.x;
                        const float4 e1 = lds4(a_rec + SM_EXTRA + RT_CHUNK * 16);
                        const float4 e2 = lds4(a_rec + SM_EXTRA + 2 * RT_CHUNK * 16);
                        const float4 e3 = lds4(a_rec + SM_EXTRA + 3 * RT_CHUNK * 16);
                        // pixel_coord = uv * radius * (1, W/H) + mean   (gaussian.wgsl:441-447; uv * radius == m)
                        const float pcx = __fadd_rn(mx, e0.y), pcy = __fadd_rn(__fmul_rn(my, e0.w), e0.z);
                        // gaussian_2d.wgsl:134-156: hu = px*T2 - T0, hv = py*T2 - T1, p = hu x hv
                        const float hux = __fsub_rn(__fmul_rn(pcx, e3.x), e1.x), huy = __fsub_rn(__fmul_rn(pcx, e3.y), e1.y),
                                    huz = __fsub_rn(__fmul_rn(pcx, e3.z), e1.z);
                        const float hvx = __fsub_rn(__fmul_rn(pcy, e3.x), e2.x), hvy = __fsub_rn(__fmul_rn(pcy, e3.y), e2.y),
                                    hvz = __fsub_rn(__fmul_rn(pcy, e3.z), e2.z);
                        const float cpx = __fsub_rn(__fmul_rn(huy, hvz), __fmul_rn(huz, hvy));
                        const float cpy = __fsub_rn(__fmul_rn(huz, hvx), __fmul_rn(hux, hvz));
                        const float cpz = __fsub_rn(__fmul_rn(hux, hvy), __fmul_rn(huy, hvx));
                        const float us = __fdiv_rn(cpx, cpz), vs = __fdiv_rn(cpy, cpz);
                        const float s3 = __fadd_rn(__fmul_rn(us, us), __fmul_rn(vs, vs));
                        const float ex = __fsub_rn(e0.y, pcx), ey = __fsub_rn(e0.z, pcy);
                        const float s2 = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)));
                        power = -__fmul_rn(0.5f, fminf(s3, s2));
                    }
                    if (power > 0.0f) continue;                      // gaussian.wgsl:468-470
                    if (BOX) edge = box && box_edge(__fdiv_rn(mx, R), __fdiv_rn(my, R));
                    q2 = lds4(a_rec + REC_Q2);
                    e = __expf(power);
                }
                if (BOX && edge) {   // the overlay colour at alpha exactly 1 (w = T) into every frame; T = 0 stops the pixel
                    if (PICK && T > best_w) { best_w = T; best_r = ps.entry(base, (a_rec - a_base) >> 4); }
                    cr = fmaf(T, 0.3f, cr); cg = fmaf(T, 1.0f, cg); cb = fmaf(T, 0.1f, cb);
                    if (AUX) {
                        dr = fmaf(T, 0.3f, dr); dg = fmaf(T, 1.0f, dg); db = fmaf(T, 0.1f, db);
                        nr = fmaf(T, 0.3f, nr); ng = fmaf(T, 1.0f, ng); nb = fmaf(T, 0.1f, nb);
                    }
                    T = 0.0f;
                    break;
                }
                const float a = fminf(e * q2.w, 0.999f);
                const float w = a * T;
                if (PICK && w > best_w) { best_w = w; best_r = ps.entry(base, (a_rec - a_base) >> 4); }
                cr = fmaf(w, q2.x, cr); cg = fmaf(w, q2.y, cg); cb = fmaf(w, q2.z, cb);
                if (AUX) {
                    const float4 ad = lds4(a_rec + SM_AUX), an = lds4(a_rec + SM_AUX + RT_CHUNK * 16);
                    dr = fmaf(w, ad.x, dr); dg = fmaf(w, ad.y, dg); db = fmaf(w, ad.z, db);
                    nr = fmaf(w, an.x, nr); ng = fmaf(w, an.y, ng); nb = fmaf(w, an.z, nb);
                }
                T = fmaf(-a, T, T);
                if (T < T_STOP) break;
            }
        }
    }
    ps.finish();
    if (!inside) return;
    if (RAW) reinterpret_cast<float4*>(out)[(size_t)py * W + px] = make_float4(cr, cg, cb, T);
    else write_pixel(out, format, (size_t)py * W + px, cr, cg, cb, T);
    if constexpr (PICK) {   // record -> global index (compact slot) -> (entity, index within its cloud), and its d
        uint4 rec = make_uint4(BGS_PICK_NONE, BGS_PICK_NONE, 0u, 0u);
        if (best_r != BGS_PICK_NONE) {
            const uint2 at = pk->locate(__ldg(pk->slot_ids + best_r));
            rec = make_uint4(at.x, at.y, __float_as_uint(best_w), __float_as_uint(__ldg(splat_d + best_r)));
        }
        pk->out[(size_t)py * W + px] = rec;
    }
    if (AUX) {
        write_pixel(out_depth, format, (size_t)py * W + px, dr, dg, db, T);
        write_pixel(out_normal, format, (size_t)py * W + px, nr, ng, nb, T);
    }
}

// The blend kernels: raster_body of one (MODE, AUX, ZTEST, BOX) and one frame kind, picked by the trailing parameter's type
// Tail: OneView (a single-view frame), ViewTable (a views frame: raster_body's VIEWS) or PickArgs / PickArgsDev (a pick
// frame: its PICK, the segments a kernel parameter or bgs_render_entities_many's device table), or SubFrames (a shutter
// frame's sub-frames: VIEWS and RAW, view i's out its slice of the sub-frame scratch).
// Every variant takes the same scalar parameters; raster_body sees null for those its variant never reads, so a variant's
// code does not depend on them.
struct OneView {};
struct SubFrames {
    ViewTable vt;
};
template <class Tail> constexpr bool IS_RAW = std::is_same<Tail, SubFrames>::value;
template <class Tail> constexpr bool IS_VIEWS = std::is_same<Tail, ViewTable>::value || IS_RAW<Tail>;
template <class Tail> constexpr bool IS_PICK = std::is_same<Tail, PickArgs>::value || std::is_same<Tail, PickArgsDev>::value;

// Minimum CTAs per SM of each variant: the most that leave it without spills (ptxas report), and for MODE 0 without aux
// the 6 its register budget was written for.
//   single view, MODE 0..2: MODE 2 with AUX and ZTEST spills at 5 (4 leave it 64 registers).
//   single view, mixed (MODE 3 / 4): ZTEST spills at 5; with AUX, MODE 4 too.
//   views: MODE 0 spills at 6; the mixed depth-tested blends, the depth-tested overlay and MODE 4's overlay at 5.  With
//     AUX: MODE 2 with ZTEST spills at 4 (3 leave it 85 registers); MODE 4, and MODE 2 and 3 with ZTEST or BOX, at 5.
//   pick: MODE 1 and 2 spill at 5 even without the depth test or the overlay; 4 leave every variant 64 registers.
template <int MODE, bool AUX, bool ZTEST, bool BOX, class Tail>
constexpr int raster_min_ctas() {
    if (IS_PICK<Tail>) return 4;
    if (IS_VIEWS<Tail> && AUX) return MODE == 2 && ZTEST ? 3 : (MODE == 4 || ((ZTEST || BOX) && MODE >= 2) ? 4 : 5);
    if (IS_VIEWS<Tail>) return (ZTEST && (MODE >= 3 || BOX)) || (BOX && MODE == 4) ? 4 : 5;
    if (MODE >= 3 && AUX) return MODE == 4 || ZTEST ? 4 : 5;
    if (MODE >= 3) return ZTEST ? 4 : 5;
    return MODE == 0 && !AUX ? 6 : (MODE == 2 && AUX && ZTEST ? 4 : 5);
}

// &tail as a T*, or null when the tail is not a T
template <class T, class Tail>
__device__ __forceinline__ const T* tail_as(const Tail& tail) {
    if constexpr (std::is_same<T, Tail>::value) return &tail;
    else return nullptr;
}
// the view table of a views or shutter frame's tail, else null
template <class Tail>
__device__ __forceinline__ const ViewTable* view_table(const Tail& tail) {
    if constexpr (IS_RAW<Tail>) return &tail.vt;
    else return tail_as<ViewTable>(tail);
}

template <int MODE, bool AUX, bool ZTEST, bool BOX, class Tail>
__global__ void __launch_bounds__(RT_THREADS, raster_min_ctas<MODE, AUX, ZTEST, BOX, Tail>())
raster_kernel(const SplatRec* __restrict__ recs, const float4* __restrict__ extra, const uint32_t* __restrict__ tile_entries,
              const uint2* __restrict__ ranges, int W, int H, int tiles_x, void* __restrict__ out, uint32_t format,
              const float4* __restrict__ aux, void* __restrict__ out_depth, void* __restrict__ out_normal,
              const uint32_t* __restrict__ truncated, const float* __restrict__ splat_d, const float* __restrict__ scene,
              size_t pitch, const unsigned char* __restrict__ kinds, const __grid_constant__ Tail tail) {
    constexpr bool VIEWS = IS_VIEWS<Tail>;   // (a views frame's size, targets and depth buffers are its view's)
    using Pick = typename std::conditional<std::is_same<Tail, PickArgsDev>::value, PickArgsDev, PickArgs>::type;
    raster_body<MODE, AUX, ZTEST, BOX, VIEWS, IS_PICK<Tail>, Pick, IS_RAW<Tail>>(
        recs, extra, tile_entries, ranges, VIEWS ? 0 : W, VIEWS ? 0 : H, VIEWS ? 0 : tiles_x, VIEWS ? nullptr : out, format,
        AUX ? aux : nullptr, AUX && !VIEWS ? out_depth : nullptr, AUX && !VIEWS ? out_normal : nullptr, truncated, splat_d,
        VIEWS ? nullptr : scene, VIEWS ? 0 : pitch, MODE >= 3 ? kinds : nullptr, view_table(tail), tail_as<Pick>(tail));
}

// the kind of each compact slot r < n_vis: its global index's segment's (overlay frames: kind | overlay << 2)
__global__ void raster_kinds_kernel(SegmentKinds sk, const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                                    unsigned char* __restrict__ out) {
    const uint32_t n_vis = ctr->n_vis;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_vis; r += gridDim.x * blockDim.x) {
        const uint32_t g = __ldg(slot_ids + r);
        uint32_t lo = 0u, hi = sk.k;   // the last j with offset <= g (SceneTable::find)
        while (hi - lo > 1u) {
            const uint32_t mid = (lo + hi) >> 1;
            if (sk.offset[mid] <= g) lo = mid; else hi = mid;
        }
        out[r] = (unsigned char)sk.kind[lo];
    }
}

// bgs_render_entities_many's: the segments are the device table's
__global__ void raster_kinds_many_kernel(SceneTableDev tab, const uint32_t* __restrict__ slot_ids,
                                         const FrameCounters* __restrict__ ctr, unsigned char* __restrict__ out) {
    const uint32_t n_vis = ctr->n_vis;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_vis; r += gridDim.x * blockDim.x)
        out[r] = (unsigned char)__ldg(tab.kinds + tab.find(__ldg(slot_ids + r)));
}

static uint32_t kinds_grid(uint32_t n_hint, int sm_count) {
    const uint32_t grid = (n_hint + 255) / 256;
    return grid < 1u ? 1u : (grid > (uint32_t)(8 * sm_count) ? (uint32_t)(8 * sm_count) : grid);
}

void launch_segment_kinds_many(const SceneTableDev& tab, const uint32_t* slot_ids, const FrameCounters* ctr, unsigned char* out,
                               uint32_t n_hint, int sm_count, cudaStream_t stream) {
    raster_kinds_many_kernel<<<kinds_grid(n_hint, sm_count), 256, 0, stream>>>(tab, slot_ids, ctr, out);
}

void launch_segment_kinds(const SegmentKinds& kinds, const uint32_t* slot_ids, const FrameCounters* ctr, unsigned char* out,
                          uint32_t n_hint, int sm_count, cudaStream_t stream) {
    raster_kinds_kernel<<<kinds_grid(n_hint, sm_count), 256, 0, stream>>>(kinds, slot_ids, ctr, out);
}

// ---- MODE 0 fast path: 2 horizontally adjacent pixels per thread -----------------------------------------
// CTA = tile, 4 warps, warp w = rows 4w..4w+3 of the tile (16x4 pixels), lane = (column pair, row).  Per
// candidate splat the record loads, the loop and dy are shared by the two pixels, and a 16-wide warp rectangle
// halves the number of (warp, splat) candidates.  Same per-pixel formulas (bit-identical coverage).
constexpr int R2_THREADS = 128;
constexpr uint32_t R2_LIST = SM_Q2 + RT_CHUNK * 16;                      // u16 [4][256]
constexpr uint32_t R2_BYTES = R2_LIST + (R2_THREADS / 32) * RT_CHUNK * 2;

__device__ __forceinline__ void store_pixel2(void* out, uint32_t format, size_t pix, bool in0, bool in1, float r0, float g0,
                                             float b0, float r1, float g1, float b1, float T0, float T1) {
    if (format >> 8) {            // premultiplied / blend-over output: the generic per-pixel path
        if (in0) write_pixel(out, format, pix, r0, g0, b0, T0);
        if (in1) write_pixel(out, format, pix + 1, r1, g1, b1, T1);
        return;
    }
    if (format == BGS_FORMAT_RGBA32F) {
        float4* o = reinterpret_cast<float4*>(out) + pix;
        if (in0) o[0] = make_float4(r0, g0, b0, 1.0f);
        if (in1) o[1] = make_float4(r1, g1, b1, 1.0f);
    } else if (format == BGS_FORMAT_RGBA16F) {
        uint2* o = reinterpret_cast<uint2*>(out) + pix;
        const uint2 p0 = pack_rgba16f(r0, g0, b0, 1.0f), p1 = pack_rgba16f(r1, g1, b1, 1.0f);
        if (in0) o[0] = p0;
        if (in1) o[1] = p1;
    } else {
        uint32_t* o = reinterpret_cast<uint32_t*>(out) + pix;
        const uint32_t p0 = pack_srgb8(r0, g0, b0, 1.0f, false), p1 = pack_srgb8(r1, g1, b1, 1.0f, false);
        // one 8-byte store where the address allows it (targets are only required to be 4-byte aligned)
        if (in0 && in1 && (reinterpret_cast<uintptr_t>(o) & 7u) == 0) *reinterpret_cast<uint2*>(o) = make_uint2(p0, p1);
        else { if (in0) o[0] = p0; if (in1) o[1] = p1; }
    }
}

// ZTEST: bgs_render_depth_test, as raster_kernel's (each pixel of the pair has its own scene depth; the warp's rectangle
// for the candidate cull is its 16x4 pixels)
template <bool CHUNKED, bool ZTEST = false>
__global__ void __launch_bounds__(R2_THREADS)
raster2_kernel(const SplatRec* __restrict__ recs, const uint32_t* __restrict__ tile_entries, const uint2* __restrict__ ranges,
               int W, int H, int tiles_x, void* __restrict__ out, uint32_t format, float4* __restrict__ state,
               unsigned char* __restrict__ tile_done, uint32_t* __restrict__ tiles_done, const uint32_t* __restrict__ truncated,
               int first, int last, const float* __restrict__ splat_d, const float* __restrict__ scene, size_t pitch) {
    __shared__ __align__(16) unsigned char s_mem[R2_BYTES + (ZTEST ? ZT_BYTES : 0)];
    constexpr uint32_t REC_D = R2_BYTES;   // ZTEST: d of the splat whose q0 record is at a, at a + REC_D
    float4* s_q0 = reinterpret_cast<float4*>(s_mem + SM_Q0);
    float4* s_uv = reinterpret_cast<float4*>(s_mem + SM_UV);
    float4* s_q2 = reinterpret_cast<float4*>(s_mem + SM_Q2);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    unsigned short* s_list = reinterpret_cast<unsigned short*>(s_mem + R2_LIST) + warp * RT_CHUNK;
    const uint32_t a_base = (uint32_t)__cvta_generic_to_shared(s_mem);
    const uint32_t a_list = a_base + R2_LIST + (uint32_t)warp * RT_CHUNK * 2u;
    int tile_x, tile_y;
    centre_out_tile((int)blockIdx.x, tiles_x, (int)gridDim.x / tiles_x, tile_x, tile_y);
    const int tile = tile_y * tiles_x + tile_x;
    const int wy0 = tile_y * TILE_PX + warp * 4;                    // this warp's 4 rows
    const int px0 = tile_x * TILE_PX + 2 * (lane & 7), py = wy0 + (lane >> 3);
    const bool in0 = px0 < W && py < H, in1 = px0 + 1 < W && py < H;
    const float fx0 = (float)px0 + 0.5f, fx1 = (float)px0 + 1.5f, fy = (float)py + 0.5f;
    uint2 range = ranges[tile];
    if (*truncated) return;              // (as raster_kernel; on a chunked frame the word also covers the earlier rounds)
    range.x = ~range.x;                  // stored as (~start, end), (0, 0) = empty (radix.cu)

    // T < T_STOP <=> pixel done; lim = 1 while alive, -1 once done (folds the "alive" test into |u| <= lim)
    float T0 = in0 ? 1.0f : 0.0f, T1 = in1 ? 1.0f : 0.0f;
    float lim0 = in0 ? 1.0f : -1.0f, lim1 = in1 ? 1.0f : -1.0f;
    float r0 = 0.f, g0 = 0.f, b0 = 0.f, r1 = 0.f, g1 = 0.f, b1 = 0.f;
    float4* st = nullptr;
    if (CHUNKED) {
        // one of several front-to-back rounds of a frame: the blend state (premultiplied rgb, transmittance) of
        // every pixel lives in `state` (tile-major, so a warp's accesses are contiguous) between rounds; since a
        // round resumes each pixel exactly where the previous one stopped, the frame is bit-identical to one round
        st = state + ((size_t)tile * R2_THREADS + t) * 2;
        if (!first) {
            const bool done = tile_done[tile] != 0;             // every pixel saturated in an earlier round
            if (!last && (done || range.x >= range.y)) return;  // nothing to blend, state unchanged
            const float4 s0 = st[0], s1 = st[1];
            r0 = s0.x; g0 = s0.y; b0 = s0.z; T0 = s0.w;
            r1 = s1.x; g1 = s1.y; b1 = s1.z; T1 = s1.w;
            lim0 = (in0 && !(T0 < T_STOP)) ? 1.0f : -1.0f;
            lim1 = (in1 && !(T1 < T_STOP)) ? 1.0f : -1.0f;
            if (done) range.y = range.x;
        }
    }
    // ZTEST: the scene depths of the two pixels (read again by every round of a chunked frame), the warp's minimum
    float zs0 = 0.0f, zs1 = 0.0f, zmin = 0.0f;
    if (ZTEST) {
        zs0 = scene_depth_at(scene, pitch, px0, py, in0);
        zs1 = scene_depth_at(scene, pitch, px0 + 1, py, in1);
        zmin = warp_min_depth(fminf(zs0, zs1));
    }
    // multi-chunk tiles (the norm on this path: heavy footprints put thousands of entries in a tile) stream their slice
    // of the sorted pair list, like raster_kernel
    __shared__ __align__(16) uint32_t s_ent[2][ENT_WORDS];
    __shared__ __align__(8) unsigned long long s_bar[2];
    PairStream ps(tile_entries, s_ent, s_bar, range, range.y > range.x && range.y - range.x > (uint32_t)RT_CHUNK);
    for (uint32_t base = range.x; base < range.y; base += RT_CHUNK, ++ps.chunk) {
        if (__syncthreads_count((lim0 > 0.f || lim1 > 0.f) ? 1 : 0) == 0) break;   // also fences smem reuse
        const uint32_t cnt = min((uint32_t)RT_CHUNK, range.y - base);
        ps.next(base);
#pragma unroll
        for (int k = 0; k < RT_CHUNK / R2_THREADS; ++k) {
            const uint32_t j = t + k * R2_THREADS;
            if (j < cnt) {
                const uint32_t r = ps.entry(base, j);
                const float4* rp = reinterpret_cast<const float4*>(recs + r);
                s_q0[j] = __ldg(rp);
                s_uv[j] = __ldg(rp + 1);
                s_q2[j] = __ldg(rp + 2);
                if (ZTEST) reinterpret_cast<float*>(s_mem + REC_D)[4 * j] = __ldg(splat_d + r);
            }
        }
        __syncthreads();
        // per-warp candidate list: splats whose bbox reaches this warp's rows (the x extent already meets the tile),
        // listed by offset of q0[j] from s_mem
        const uint32_t nl = !__any_sync(0xffffffffu, lim0 > 0.f || lim1 > 0.f) ? 0u : compact_candidates(cnt, s_list, 0u, [&](uint32_t j) {
            const uint32_t by = __float_as_uint(s_uv[j].w);
            const bool hit = !((int)(by >> 16) < wy0 || (int)(by & 0xFFFFu) > wy0 + 3);
            return ZTEST ? hit && !(reinterpret_cast<const float*>(s_mem + REC_D)[4 * j] < zmin) : hit;
        });
        if (lim0 > 0.f || lim1 > 0.f) {
            const uint32_t a_end = a_list + nl * 2u;
            for (uint32_t a_it = a_list; a_it != a_end; a_it += 2u) {
                const uint32_t a_rec = a_base + lds_u16(a_it);
                const float4 q0 = lds4(a_rec);
                const float2 q1 = lds2(a_rec + REC_UV);
                const float2 uva = quad_uv(fx0, fy, q0, q1), uvb = quad_uv(fx1, fy, q0, q1);   // (dy is computed once)
                bool ca = fabsf(uva.x) <= lim0 && fabsf(uva.y) <= lim0;
                bool cb = fabsf(uvb.x) <= lim1 && fabsf(uvb.y) <= lim1;
                if (ZTEST) {
                    const float d = lds_f32(a_rec + REC_D);
                    ca = ca && d >= zs0;
                    cb = cb && d >= zs1;
                }
                if (!(ca || cb)) continue;
                const float4 q2 = lds4(a_rec + REC_Q2);
                if (ca) {
                    float e;
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(__fmaf_rn(uva.y, uva.y, __fmul_rn(uva.x, uva.x)) * -6.492127684f));
                    const float a = fminf(e * q2.w, 0.999f);
                    const float w = a * T0;
                    r0 = fmaf(w, q2.x, r0); g0 = fmaf(w, q2.y, g0); b0 = fmaf(w, q2.z, b0);
                    T0 = fmaf(-a, T0, T0);
                    if (T0 < T_STOP) lim0 = -1.0f;
                }
                if (cb) {
                    float e;
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(__fmaf_rn(uvb.y, uvb.y, __fmul_rn(uvb.x, uvb.x)) * -6.492127684f));
                    const float a = fminf(e * q2.w, 0.999f);
                    const float w = a * T1;
                    r1 = fmaf(w, q2.x, r1); g1 = fmaf(w, q2.y, g1); b1 = fmaf(w, q2.z, b1);
                    T1 = fmaf(-a, T1, T1);
                    if (T1 < T_STOP) lim1 = -1.0f;
                }
                if (!(lim0 > 0.f || lim1 > 0.f)) break;
            }
        }
    }
    ps.finish();
    if (CHUNKED && !last) {
        st[0] = make_float4(r0, g0, b0, T0);
        st[1] = make_float4(r1, g1, b1, T1);
        if (__syncthreads_count((lim0 > 0.f || lim1 > 0.f) ? 1 : 0) == 0 && t == 0) {
            tile_done[tile] = 1;
            atomicAdd(tiles_done, 1u);
        }
        return;
    }
    if (!(in0 || in1)) return;
    store_pixel2(out, format, (size_t)py * W + px0, in0, in1, r0, g0, b0, r1, g1, b1, T0, T1);
}

// The blend kernels of one Tail, indexed mode + 5 (box + 2 (ztest + 2 aux)) (pick and shutter frames have no aux variants)
template <class Tail, int... I>
const auto* blend_kernels(std::integer_sequence<int, I...>) {
    static void (*const table[])(const SplatRec*, const float4*, const uint32_t*, const uint2*, int, int, int, void*, uint32_t,
                                 const float4*, void*, void*, const uint32_t*, const float*, const float*, size_t,
                                 const unsigned char*, const Tail) = {
        raster_kernel<I % 5, I >= 20, (I / 10) % 2 != 0, (I / 5) % 2 != 0, Tail>...};
    return table;
}

template <class Tail>
void launch_blend(const BlendArgs& a, uint32_t grid, const Tail& tail, cudaStream_t stream) {
    static const auto* const kernels = blend_kernels<Tail>(std::make_integer_sequence<int, IS_PICK<Tail> || IS_RAW<Tail> ? 20 : 40>());
    const int i = a.mode + 5 * ((a.box ? 1 : 0) + 2 * ((a.scene ? 1 : 0) + 2 * (a.aux ? 1 : 0)));
    kernels[i]<<<grid, RT_THREADS, 0, stream>>>(
        a.recs, a.extra, a.tile_entries, a.ranges, a.W, a.H, a.tiles_x, a.out, a.format, a.aux, a.out_depth, a.out_normal,
        a.truncated, a.splat_d, a.scene, a.pitch, a.kinds, tail);
}

void launch_raster(const BlendArgs& a, cudaStream_t stream) {
    if (a.views && a.raw) {
        launch_blend(a, a.views->tile0[a.views->v], SubFrames{*a.views}, stream);
    } else if (a.views) {
        launch_blend(a, a.views->tile0[a.views->v], *a.views, stream);
    } else if (a.pick) {
        launch_blend(a, (uint32_t)(a.tiles_x * a.tiles_y), *a.pick, stream);
    } else if (a.pick_dev) {
        launch_blend(a, (uint32_t)(a.tiles_x * a.tiles_y), *a.pick_dev, stream);
    } else if (a.mode == 0 && !a.aux && !a.box && a.large_footprints) {
        // the 2-pixels-per-thread variant wins when splats cover many tiles each and loses when most splats are a few
        // pixels (more of its lanes then idle at the tile's splat boundaries)
        auto* kernel = a.scene ? raster2_kernel<false, true> : raster2_kernel<false, false>;
        kernel<<<a.tiles_x * a.tiles_y, R2_THREADS, 0, stream>>>(
            a.recs, a.tile_entries, a.ranges, a.W, a.H, a.tiles_x, a.out, a.format, nullptr, nullptr, nullptr, a.truncated, 1, 1,
            a.splat_d, a.scene, a.pitch);
    } else {
        launch_blend(a, (uint32_t)(a.tiles_x * a.tiles_y), OneView{}, stream);
    }
}

// One front-to-back round of a chunked frame (quad-uv records only); see raster2_kernel.
void launch_raster_round(const BlendArgs& a, float4* state, unsigned char* tile_done, uint32_t* tiles_done, int first, int last,
                         cudaStream_t stream) {
    (a.scene ? raster2_kernel<true, true> : raster2_kernel<true, false>)<<<a.tiles_x * a.tiles_y, R2_THREADS, 0, stream>>>(
        a.recs, a.tile_entries, a.ranges, a.W, a.H, a.tiles_x, a.out, a.format, state, tile_done, tiles_done, a.truncated, first,
        last, a.splat_d, a.scene, a.pitch);
}

}  // namespace bgs
