// project.cu -- stage 3: per-gaussian 3D->2D covariance projection + SH colour (degree 0..3), run
// ONCE per visible gaussian (the reference runs it 4x per gaussian in its vertex stage:
// src/render/gaussian.wgsl:185-436).
//
// Record r of n_vis is the gaussian id the index list gives for r (project_kernel's `by_slot`):
//  * compact frames (the default): r is a compact slot, id = slot_ids[r] (ascending gaussian index, as key-gen
//    compacted them).  The projection runs beside the depth sort, whose payload is that slot: binning reads the
//    record of rank k at recs[sorted slot of k];
//  * BGS_FLAG_SORT_ALL: r is a front-to-back rank (0 = nearest), id = sorted_ids[n_vis-1-r] (the sort is far->near
//    like the reference's, src/sort/radix.wgsl).
// Either way: gather the gaussian's block (cloud_layout.cuh) -> write one 48 B SplatRec at recs[r]
// (coalesced), which is all the tile stages read.
//
// project_one is the vertex stage's dispatch: frustum and draw-mode test, cutoff, then the record of the splat's
// geometry (3DGS USE_AABB conic, 3DGS USE_OBB, 2DGS surfel) and its colour source (SH, Depth, Normal, Position).
// Geometry (centre, OBB uv rows, pixel bbox) is bit-exact vs the oracle: compiled -fmad=false.
#include "project_math.cuh"
#include "entry_src.cuh"
#include "launch.cuh"

namespace bgs {

__constant__ float c_shc[16] = {   // src/material/spherical_harmonics.wgsl:3-20
    0.28209479177387814f, -0.4886025119029199f, 0.4886025119029199f, -0.4886025119029199f,
    1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
    0.5462742152960396f, -0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
    0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

// colour path only (compared under tolerance): one rsqrt.approx (2 ulp) instead of an IEEE sqrt + three divisions
__device__ __forceinline__ void normalize3(const float a[3], float out[3]) {
    const float inv = rsqrtf((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]);
    out[0] = a[0] * inv; out[1] = a[1] * inv; out[2] = a[2] * inv;
}
__device__ __forceinline__ float dot3(const float a[3], const float b[3]) {
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2];
}
// spherical_harmonics.wgsl:22-32; no clamp on either side
// (colour is compared under tolerance, not bit-exactly: fast pow = ex2(2.4 * lg2 x), ~1e-6 relative)
__device__ __forceinline__ float srgb_to_linear(float v) {
    if (v <= 0.04045f) return v * (1.0f / 12.92f);
    return __powf((v + 0.055f) * (1.0f / 1.055f), 2.4f);
}
__device__ __forceinline__ uint32_t pack_bbox(float lo, float hi) {
    return (uint32_t)(int)lo | ((uint32_t)(int)hi << 16);
}
constexpr uint32_t BBOX_EMPTY = 1u;   // lo = 1, hi = 0

// conservative pixel bbox of |fx - cx| <= hx, |fy - cy| <= hy (this repo's a7 rule; see oracle)
__device__ __forceinline__ void make_bbox(float cx, float cy, float hx, float hy, int Wi, int Hi,
                                          uint32_t& bx, uint32_t& by) {
    bx = BBOX_EMPTY; by = BBOX_EMPTY;
    if (!(hx >= 0.0f) || !(hy >= 0.0f) || !(cx == cx) || !(cy == cy)) return;
    const float sx = hx * 1.0e-3f + 1.0e-2f, sy = hy * 1.0e-3f + 1.0e-2f;
    float x0 = ceilf((cx - hx) - (0.5f + sx));
    float x1 = floorf((cx + hx) - (0.5f - sx));
    float y0 = ceilf((cy - hy) - (0.5f + sy));
    float y1 = floorf((cy + hy) - (0.5f - sy));
    if (!(x0 <= x1) || !(y0 <= y1)) return;
    x0 = fmaxf(x0, 0.0f); y0 = fmaxf(y0, 0.0f);
    x1 = fminf(x1, (float)(Wi - 1)); y1 = fminf(y1, (float)(Hi - 1));
    if (!(x0 <= x1) || !(y0 <= y1)) return;
    bx = pack_bbox(x0, x1); by = pack_bbox(y0, y1);
}

// Attributes come from the cloud's gaussian-major blocks (cloud_layout.cuh), so the random gather of a visible splat
// touches exactly its own line(s) instead of 3-4 partially used ones of the reference's planes.
//
// A warp gathers the blocks of 32 consecutive entries of the index list into its own shared-memory stage with
// coalesced 16 B asynchronous copies (cp.async.cg: no staging registers, L1 bypassed, every line is used once; the
// source's copy, entry_src.cuh).  NP = CH (the whole block) when the colour source reads the SH coefficients, else GEO
// pieces: position, rotation, scale and opacity (f32: plus the first SH piece, which shares scale_opacity's 32 B
// sector).  Piece p of entry g sits at 16 B unit g * CH + stage_slot<CH>(p, g): the eight lanes of a quarter warp that
// read the same piece of their own entries hit eight different 16 B bank groups, and so do the copies' stores.

// entry g's attributes out of a stage, the S_d SH floats into sh (the covariance layout's record arrives in q and so as
// its lanes fall)
template <bool F16, uint32_t D>
struct Attr;
template <uint32_t D>
struct Attr<false, D> {
    static constexpr CloudLayout L = CloudLayout::F32;
    static constexpr int CH = chunks(L, D), GEO = 4;
    __device__ static float4 load(const uint4* stage, int g, float* sh, float q[4], float so[4], bool need_sh, uint32_t&) {
        auto piece = [&](int p) {
            const uint4 v = stage[g * CH + stage_slot<CH>(p, g)];
            return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w));
        };
        const float4 p = piece(POS_CHUNK), r = piece(SECOND_CHUNK), s = piece(SO_CHUNK);
        q[0] = r.x; q[1] = r.y; q[2] = r.z; q[3] = r.w;
        so[0] = s.x; so[1] = s.y; so[2] = s.z; so[3] = s.w;
        if (need_sh) {
#pragma unroll
            for (int i = 0; i < (int)sh_chunks(L, D); ++i) {
                const float4 v = piece(sh_first(L) + i);
                sh[4 * i] = v.x; sh[4 * i + 1] = v.y; sh[4 * i + 2] = v.z; sh[4 * i + 3] = v.w;
            }
        }
        return p;
    }
};
template <uint32_t D>
struct Attr<true, D> {
    static constexpr CloudLayout L = CloudLayout::F16;
    static constexpr int CH = chunks(L, D), GEO = 2;
    static constexpr int FULL = (int)sh_floats(D) / 8;   // SH chunks of 4 words; below degree 3 a last one of 2 words
    __device__ static float4 load(const uint4* stage, int g, float* sh, float q[4], float so[4], bool need_sh,
                                  uint32_t& op_bits) {
        auto piece = [&](int p) { return stage[g * CH + stage_slot<CH>(p, g)]; };
        const uint4 pw = piece(POS_CHUNK), w = piece(SECOND_CHUNK);
        op_bits = w.w & 0xFFFFu;
        second_lanes(w.x, w.y, q);
        second_lanes(w.z, w.w, so);
        if (need_sh) {
#pragma unroll
            for (int i = 0; i < FULL; ++i) {
                const uint4 v = piece(sh_first(L) + i);
                sh[8 * i] = half_lo(v.x); sh[8 * i + 1] = half_hi(v.x); sh[8 * i + 2] = half_lo(v.y); sh[8 * i + 3] = half_hi(v.y);
                sh[8 * i + 4] = half_lo(v.z); sh[8 * i + 5] = half_hi(v.z); sh[8 * i + 6] = half_lo(v.w); sh[8 * i + 7] = half_hi(v.w);
            }
            if constexpr (sh_floats(D) % 8 != 0) {
                const uint4 v = piece(sh_first(L) + FULL);
                sh[8 * FULL] = half_lo(v.x); sh[8 * FULL + 1] = half_hi(v.x);
                sh[8 * FULL + 2] = half_lo(v.y); sh[8 * FULL + 3] = half_hi(v.y);
            }
        }
        return make_float4(__uint_as_float(pw.x), __uint_as_float(pw.y), __uint_as_float(pw.z), __uint_as_float(pw.w));
    }
};

// upload-time repack of the planes into gaussian-major blocks (one thread per 16 B chunk; coalesced both ways)
template <CloudLayout L, uint32_t D>
__device__ __forceinline__ void repack_chunk(const CloudPlanes<const uint4>& planes, uint32_t n, uint4* __restrict__ blocks,
                                             const uint4* __restrict__ tt) {
    constexpr uint32_t CH = chunks(L, D);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * CH) return;
    const uint4* src = planes.unit<L, D>((uint32_t)(i % CH), i / CH, tt);
    blocks[i] = src ? __ldg(src) : make_uint4(0u, 0u, 0u, 0u);
}
template <CloudLayout L, uint32_t D>
__global__ void repack_kernel(CloudPlanes<const uint4> planes, uint32_t n, uint4* __restrict__ blocks) {
    repack_chunk<L, D>(planes, n, blocks, nullptr);
}
// the 4D layout's, which also reads the timestamp-timescale plane
__global__ void repack_4d_kernel(CloudPlanes<const uint4> planes, uint32_t n, uint4* __restrict__ blocks,
                                 const uint4* __restrict__ tt) {
    repack_chunk<CloudLayout::F32x4D, SH_DEGREE_MAX>(planes, n, blocks, tt);
}
void launch_repack(CloudLayout layout, uint32_t sh_degree, const void* sh, const void* rot, const void* so, const void* tt,
                   uint32_t n, CloudView cloud, cudaStream_t stream) {
    const CloudPlanes<const uint4> planes{reinterpret_cast<const uint4*>(cloud.pos), static_cast<const uint4*>(sh),
                                          static_cast<const uint4*>(rot), static_cast<const uint4*>(so)};
    const uint32_t grid = (uint32_t)(((size_t)n * cloud.chunks + 255) / 256);
    with_layout_degree(layout, sh_degree, [&](auto L, auto D) {
        if constexpr (is_4d(decltype(L)::value))
            repack_4d_kernel<<<grid, 256, 0, stream>>>(planes, n, cloud.blocks, static_cast<const uint4*>(tt));
        else
            repack_kernel<decltype(L)::value, decltype(D)::value><<<grid, 256, 0, stream>>>(planes, n, cloud.blocks);
    });
}

// RasterizeMode::Depth (gaussian.wgsl:329-349): min distance from sorted[N-1], max from sorted[1] of the
// reference's FULL sorted buffer (culled entries keyed all-ones sit at its end, in index order) -- literal,
// including the [1] (not [0]) and the fact that the "nearest" entry is a culled gaussian whenever one exists.
template <class Src>
__device__ __forceinline__ void depth_range_body(const Src& src, uint32_t n, const uint32_t* __restrict__ sorted_payload,
                                                 const uint32_t* __restrict__ slot_ids, FrameCounters* __restrict__ ctr) {
    if (threadIdx.x != 0 || blockIdx.x != 0 || n < 2u) return;
    const uint32_t n_vis = ctr->n_vis, n_sorted = ctr->n_sort;
    auto id_at = [&](uint32_t i) { const uint32_t p = sorted_payload[i]; return slot_ids ? slot_ids[p] : p; };
    uint32_t first, last;
    if (n_sorted == n) {                       // SORT_ALL: the full buffer is materialised
        first = id_at(1u); last = id_at(n - 1u);
    } else {
        const uint32_t cmin = 0xFFFFFFFFu - ctr->culled_min_inv, cmax = ctr->culled_max_p1 - 1u;
        first = n_vis >= 2u ? id_at(1u) : cmin;            // n_vis == 0 draws nothing: value irrelevant
        last = (n - n_vis) >= 1u ? cmax : id_at(n - 1u);
    }
    auto dist = [&](uint32_t id) {
        const uint32_t j = src.seg(id);
        const FrameConsts& fc = src.fc(j);
        const float4 p = *src.pos_at(j, id);
        float pw[4];
        mat4_point(fc.model, p.x, p.y, p.z, pw);
        return sqrtf(cam_dist2(fc, pw));
    };
    ctr->depth_min = dist(last);
    ctr->depth_max = dist(first);
}

__global__ void depth_range_kernel(const float4* __restrict__ pos, uint32_t n, const uint32_t* __restrict__ sorted_payload,
                                   const uint32_t* __restrict__ slot_ids /* null: payload is the gaussian index */,
                                   FrameCounters* __restrict__ ctr, FrameConsts fc) {
    depth_range_body(OneCloud{pos, fc}, n, sorted_payload, slot_ids, ctr);
}

// bgs_render_scene (compact frames only: it refuses SORT_ALL); the SORT_ALL branch takes the compact one's ends when
// every gaussian is visible
__global__ void depth_range_scene_kernel(SceneTable tab, const uint32_t* __restrict__ sorted_payload,
                                         const uint32_t* __restrict__ slot_ids, FrameCounters* __restrict__ ctr) {
    depth_range_body(SceneSrc{tab}, tab.n_total, sorted_payload, slot_ids, ctr);
}

// gaussian.wgsl:228-232: cutoff = sqrt(max(9 + 2 ln(opacity), 1e-6)) (fixed-series ln, see project_math.cuh)
__device__ __forceinline__ float adaptive_cutoff(float opacity) {
    const float a = 9.0f + 2.0f * det_ln(opacity);
    return sqrtf(a > 0.000001f ? a : 0.000001f);
}
// f16 clouds: the adaptive cutoff depends on the 16-bit opacity alone -> a 65536-entry table built once per context
// by this very function (bit-identical to evaluating it in place, ~70 f64 instructions cheaper per gaussian)
__global__ void cutoff_table_kernel(float* __restrict__ tab) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h < 65536u) tab[h] = adaptive_cutoff(__half2float(__ushort_as_half((unsigned short)h)));
}
void launch_cutoff_table(float* tab, cudaStream_t stream) { cutoff_table_kernel<<<256, 256, 0, stream>>>(tab); }

// gaussian.wgsl:228-232: the quad's extent in standard deviations; with OPACITY_ADAPTIVE_RADIUS, f16 clouds read it
// from the table of their 16-bit opacity
template <bool F16>
__device__ __forceinline__ float splat_cutoff(const FrameConsts& fc, float opacity, const float* __restrict__ cutoff_tab,
                                              uint32_t op_bits) {
    if (!fc.adaptive) return 3.0f;
    if constexpr (F16) return __ldg(cutoff_tab + op_bits);
    else return adaptive_cutoff(opacity);
}

// helpers.wgsl:137-158 as (row, col); the quaternion is NOT normalised
__device__ __forceinline__ void rotation_rows(const float q[4], float Rm[3][3]) {
    const float qr = q[0], x = q[1], y = q[2], z = q[3];
    Rm[0][0] = 1.0f - 2.0f * (y * y + z * z);
    Rm[1][0] = 2.0f * (x * y - qr * z);
    Rm[2][0] = 2.0f * (x * z + qr * y);
    Rm[0][1] = 2.0f * (x * y + qr * z);
    Rm[1][1] = 1.0f - 2.0f * (x * x + z * z);
    Rm[2][1] = 2.0f * (y * z - qr * x);
    Rm[0][2] = 2.0f * (x * z - qr * y);
    Rm[1][2] = 2.0f * (y * z + qr * x);
    Rm[2][2] = 1.0f - 2.0f * (x * x + y * y);
}

// gaussian_3d.wgsl:49-72: the world-space covariance T Sigma T^t, Sigma = M^t M, M = S R, T = the model 3x3, as its six
// entries (WGSL [col][row] order)
__device__ __forceinline__ void sigma3d(const FrameConsts& fc, const float A[3][3], const float Rm[3][3], const float sc[3],
                                        const float q[4], const float so[4], float c3[6]) {
    if (fc.cov_pre) {
        // PRECOMPUTE_COVARIANCE_3D (gaussian_3d.wgsl:78-79, planar.wgsl:133-152): the decoded record goes straight into
        // cov2d -- no global_scale, no model 3x3.  It arrives in the plane slots it occupies: q = c0..c3, so = c4, c5,
        // opacity, opacity
        c3[0] = q[0]; c3[1] = q[1]; c3[2] = q[2]; c3[3] = q[3]; c3[4] = so[0]; c3[5] = so[1];
        return;
    }
    float M[3][3], Sg[3][3], X[3][3], TS[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) M[i][j] = sc[i] * Rm[i][j];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Sg[i][j] = (M[0][i] * M[0][j] + M[1][i] * M[1][j]) + M[2][i] * M[2][j];
    // identity model: T Sigma T^t == Sigma bit for bit as long as every entry of Sigma is finite and NON-ZERO
    // (x*1 + y*0 + z*0 then only ever adds +-0 to a non-zero value); zero entries (axis-aligned splats) keep
    // the multiply so that even the sign of a zero matches the oracle
    const float mn = fminf(fminf(fminf(fabsf(Sg[0][0]), fabsf(Sg[0][1])), fminf(fabsf(Sg[0][2]), fabsf(Sg[1][1]))),
                           fminf(fabsf(Sg[1][2]), fabsf(Sg[2][2])));
    const float mx = fmaxf(fmaxf(fmaxf(fabsf(Sg[0][0]), fabsf(Sg[0][1])), fmaxf(fabsf(Sg[0][2]), fabsf(Sg[1][1]))),
                           fmaxf(fabsf(Sg[1][2]), fabsf(Sg[2][2])));
    if (fc.model_identity && mn > 0.0f && mx < __uint_as_float(0x7F800000u) && Sg[0][0] == Sg[0][0] &&
        Sg[0][1] == Sg[0][1] && Sg[0][2] == Sg[0][2] && Sg[1][1] == Sg[1][1] && Sg[1][2] == Sg[1][2] && Sg[2][2] == Sg[2][2]) {
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) TS[i][j] = Sg[i][j];
    } else {
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) X[i][j] = (A[i][0] * Sg[0][j] + A[i][1] * Sg[1][j]) + A[i][2] * Sg[2][j];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) TS[i][j] = (X[i][0] * A[j][0] + X[i][1] * A[j][1]) + X[i][2] * A[j][2];
    }
    c3[0] = TS[0][0]; c3[1] = TS[1][0]; c3[2] = TS[2][0]; c3[3] = TS[1][1]; c3[4] = TS[2][1]; c3[5] = TS[2][2];
}

// helpers.wgsl:8-67: the screen-space covariance [a b; b c] (+0.3 on the diagonal) of the splat at pw, its determinant
// and its eigenvalues mid +- term (l1 = the larger)
struct Cov2d {
    float a, b, c, det, mid, term, l1;
};
__device__ __forceinline__ Cov2d cov2d(const FrameConsts& fc, const float pw[3], const float c3[6]) {
    const float Vrk[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
    float tv[4];
    mat4_point(fc.view_from_world, pw[0], pw[1], pw[2], tv);
    const float fx = fc.p00 * fc.W, fy = fc.p11 * fc.H;
    const float sz = 1.0f / (tv[2] * tv[2]);
    const float J00 = fx / tv[2], J20 = -(fx * tv[0]) * sz;
    const float J11 = -fy / tv[2], J21 = (fy * tv[1]) * sz;
    float Tm[3][2];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float v0 = fc.view_from_world[i * 4 + 0], v1 = fc.view_from_world[i * 4 + 1],
                    v2 = fc.view_from_world[i * 4 + 2];
        Tm[i][0] = v0 * J00 + v2 * J20;
        Tm[i][1] = v1 * J11 + v2 * J21;
    }
    float Y[3][2];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int b = 0; b < 2; ++b) Y[i][b] = (Vrk[i][0] * Tm[0][b] + Vrk[i][1] * Tm[1][b]) + Vrk[i][2] * Tm[2][b];
    Cov2d v;
    v.a = ((Tm[0][0] * Y[0][0] + Tm[1][0] * Y[1][0]) + Tm[2][0] * Y[2][0]) + 0.3f;
    v.b = (Tm[0][1] * Y[0][0] + Tm[1][1] * Y[1][0]) + Tm[2][1] * Y[2][0];
    v.c = ((Tm[0][1] * Y[0][1] + Tm[1][1] * Y[1][1]) + Tm[2][1] * Y[2][1]) + 0.3f;
    v.det = v.a * v.c - v.b * v.b;
    v.mid = 0.5f * (v.a + v.c);
    v.term = sqrtf(fmaxf(0.0f, v.mid * v.mid - v.det));
    v.l1 = v.mid + v.term;
    return v;
}

// helpers.wgsl:69-79 + gaussian.wgsl:299-309 (USE_AABB): a square of half-side cutoff * sqrt(l1) and the conic
// record: ux, uy, vx = conic.x, .y, .z; vy = the quad's half-side (half-pixels)
__device__ __forceinline__ void aabb_record(const FrameConsts& fc, const Cov2d& v, float cutoff, SplatRec& rec) {
    const float l2 = fmaxf(v.mid - v.term, 0.0f);
    const float Rq = cutoff * fmaxf(sqrtf(v.l1), sqrtf(l2));
    const float dinv = 1.0f / v.det;
    rec.ux = v.c * dinv; rec.uy = -v.b * dinv; rec.vx = v.a * dinv; rec.vy = Rq;
    const float h = 0.5f * Rq;
    make_bbox(rec.cx, rec.cy, h, h, fc.Wi, fc.Hi, rec.bx, rec.by);
}

// helpers.wgsl:81-119 (USE_OBB): the rows of the pixel-offset -> quad-uv map along the eigenvectors, scaled by
// cutoff * the axis lengths; no bbox when the map is NaN (b = 0 and a = c)
__device__ __forceinline__ void obb_record(const FrameConsts& fc, const Cov2d& v, float cutoff, SplatRec& rec) {
    const float a = v.a, b = v.b, c = v.c;
    const float aa = (a - c) * (a - c);
    const float bb = sqrtf(aa + (4.0f * b) * b);
    const float major = sqrtf(((a + c) + bb) * 0.5f);
    const float minor = sqrtf(((a + c) - bb) * 0.5f);
    const float Bx = cutoff * major, By = cutoff * minor;
    const float evx = -b, evy = v.l1 - a;
    const float el = sqrtf(evx * evx + evy * evy);
    const float e1x = evx / el, e1y = evy / el;
    const float e2x = e1y, e2y = -e1x;
    rec.ux = (2.0f * e1x) / Bx; rec.uy = (-2.0f * e1y) / Bx;
    rec.vx = (2.0f * e2x) / By; rec.vy = (-2.0f * e2y) / By;
    const float hx = 0.5f * (fabsf(e1x) * Bx + fabsf(e2x) * By);
    const float hy = 0.5f * (fabsf(e1y) * Bx + fabsf(e2y) * By);
    if (rec.ux == rec.ux && rec.uy == rec.uy && rec.vx == rec.vx && rec.vy == rec.vy)
        make_bbox(rec.cx, rec.cy, hx, hy, fc.Wi, fc.Hi, rec.bx, rec.by);
}

// 2DGS surfel: gaussian_2d.wgsl:77-132 (homography) + :49-75 (quad).  The record is an OBB one with e1 = (1, 0),
// e2 = (0, 1); with USE_AABB the blend evaluates the ray-splat intersection from the homography rows in extra[4 r..]
__device__ __forceinline__ void surfel_record(const FrameConsts& fc, const float A[3][3], const float Rm[3][3],
                                              const float sc[3], const float pw[3], float cutoff, uint32_t r,
                                              float4* __restrict__ extra, SplatRec& rec) {
    const float W = fc.W, H = fc.H;
    float L[3][2];   // first two columns of A * R_std * S, R_std = transpose(Rm)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const float rc[3] = {Rm[j][0] * sc[j], Rm[j][1] * sc[j], Rm[j][2] * sc[j]};
#pragma unroll
        for (int i = 0; i < 3; ++i) L[i][j] = (A[i][0] * rc[0] + A[i][1] * rc[1]) + A[i][2] * rc[2];
    }
    float G[3][4];
    mat4_dir(fc.clip_from_world, L[0][0], L[1][0], L[2][0], G[0]);
    mat4_dir(fc.clip_from_world, L[0][1], L[1][1], L[2][1], G[1]);
    mat4_point(fc.clip_from_world, pw[0], pw[1], pw[2], G[2]);
    const float fxk = fc.p00 * W / 2.0f, fyk = fc.p11 * H / 2.0f;     // helpers.wgsl:122-135
    const float cxk = (W - 1.0f) / 2.0f, cyk = (H - 1.0f) / 2.0f;
    float T0[3], T1[3], T2[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        T0[j] = fxk * G[j][0] + cxk * G[j][3];
        T1[j] = fyk * G[j][1] + cyk * G[j][3];
        T2[j] = G[j][3];
    }
    const float c2 = cutoff * cutoff;
    const float test[3] = {c2, c2, -1.0f};
    const float tt[3] = {test[0] * T2[0], test[1] * T2[1], test[2] * T2[2]};
    const float d = dot3(tt, T2);
    if (fabsf(d) < 1.0e-4f) return;
    const float inv = 1.0f / d;
    const float f[3] = {inv * test[0], inv * test[1], inv * test[2]};
    const float t02[3] = {T0[0] * T2[0], T0[1] * T2[1], T0[2] * T2[2]};
    const float t12[3] = {T1[0] * T2[0], T1[1] * T2[1], T1[2] * T2[2]};
    const float mean0 = dot3(f, t02), mean1 = dot3(f, t12);
    const float f0[3] = {f[0] * T0[0], f[1] * T0[1], f[2] * T0[2]};
    const float f1[3] = {f[0] * T1[0], f[1] * T1[1], f[2] * T1[2]};
    const float ex = mean0 * mean0 - dot3(f0, T0);
    const float ey = mean1 * mean1 - dot3(f1, T1);
    if (ex < 1.0e-4f || ey < 1.0e-4f) return;
    const float Rq = fmaxf(fmaxf(sqrtf(ex), sqrtf(ey)), cutoff * 0.707106f);
    rec.ux = 2.0f / Rq; rec.uy = 0.0f; rec.vx = 0.0f; rec.vy = -2.0f / Rq;
    const float h = 0.5f * Rq;
    if (Rq == Rq) make_bbox(rec.cx, rec.cy, h, h, fc.Wi, fc.Hi, rec.bx, rec.by);
    if (fc.aabb && extra != nullptr) {
        float4* e = extra + (size_t)r * 4;
        e[0] = make_float4(Rq, mean0, mean1, W / H);
        e[1] = make_float4(T0[0], T0[1], T0[2], 0.0f);
        e[2] = make_float4(T1[0], T1[1], T1[2], 0.0f);
        e[3] = make_float4(T2[0], T2[1], T2[2], 0.0f);
    }
}

// The SH-3 basis of the camera ray in the splat's model frame (gaussian.wgsl:166-183,406-416, spherical_harmonics.wgsl:
// 34-68), the SH constants folded in (16 multiplies instead of 48)
__device__ __forceinline__ void sh_basis(const FrameConsts& fc, const float A[3][3], const float pw[3], float basis[16]) {
    const float dlt[3] = {pw[0] - fc.cam[0], pw[1] - fc.cam[1], pw[2] - fc.cam[2]};
    float dw[3], loc[3], dl[3];
    normalize3(dlt, dw);
    if (fc.model_identity) {     // the normalised model columns are the unit axes
        loc[0] = dw[0]; loc[1] = dw[1]; loc[2] = dw[2];
    } else {
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
            const float col[3] = {A[0][cc], A[1][cc], A[2][cc]};
            float bn[3];
            normalize3(col, bn);
            loc[cc] = dot3(bn, dw);
        }
    }
    normalize3(loc, dl);
    const float x = dl[0], y = dl[1], z = dl[2];
    const float xx = x * x, yy = y * y, zz = z * z;
    basis[0] = 1.0f;
    basis[1] = y; basis[2] = z; basis[3] = x;
    basis[4] = x * y; basis[5] = y * z; basis[6] = (2.0f * zz - xx) - yy;
    basis[7] = x * z; basis[8] = xx - yy;
    basis[9] = y * (3.0f * xx - yy);
    basis[10] = (x * y) * z;
    basis[11] = y * ((4.0f * zz - xx) - yy);
    basis[12] = z * ((2.0f * zz - 3.0f * xx) - 3.0f * yy);
    basis[13] = x * ((4.0f * zz - xx) - yy);
    basis[14] = z * (xx - yy);
    basis[15] = x * (xx - 3.0f * yy);
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) basis[kk] *= c_shc[kk];
}

// RasterizeMode::Color: the SH colour seen along the camera ray in the splat's model frame, over the K_d bands of degree
// D (spherical_harmonics.wgsl:34-68 keeps the bands its SH_COEFF_COUNT holds); sh holds S_d floats
template <uint32_t D>
__device__ __forceinline__ void sh_colour(const FrameConsts& fc, const float A[3][3], const float pw[3], const float* sh,
                                          float rgb[3]) {
    float basis[16];
    sh_basis(fc, A, pw, basis);
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) {
        float acc = 0.5f;
#pragma unroll
        for (int kk = 0; kk < (int)sh_bands(D); ++kk) acc = fmaf(sh[3 * kk + cc], basis[kk], acc);   // colour: FMA is fine
        rgb[cc] = acc;
    }
    if (fc.color_space == 0u) {
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) rgb[cc] = srgb_to_linear(rgb[cc]);
    }
}

// RasterizeMode::Depth: material/depth.wgsl:3-11 over the range (depth_min, depth_max) that range() reads
template <class Range>
__device__ __forceinline__ void depth_colour_over(const FrameConsts& fc, Range range, const float pw[3], float rgb[3]) {
    if (fc.n_cloud < 2u) return;   // the reference reads sorted[1]: undefined for a 1-gaussian cloud (oracle: black)
    const float depth = sqrtf(cam_dist2(fc, pw));
    const float2 dr = range();
    const float dmin = dr.x, dmax = dr.y;
    float nd = (depth - dmin) / (dmax - dmin);
    nd = fminf(fmaxf(nd, 0.0f), 1.0f);   // fmin/fmax ignore a NaN operand, like the oracle's
    float t1 = (nd - 0.5f) / (1.0f - 0.5f); t1 = fminf(fmaxf(t1, 0.0f), 1.0f);
    float t2 = (nd - 0.0f) / (0.5f - 0.0f); t2 = fminf(fmaxf(t2, 0.0f), 1.0f);
    rgb[0] = t1 * t1 * (3.0f - 2.0f * t1);
    rgb[1] = 1.0f - fabsf(nd - 0.5f) * 2.0f;
    rgb[2] = 1.0f - t2 * t2 * (3.0f - 2.0f * t2);
}
// ... over depth_range_kernel's [depth_min, depth_max]
__device__ __forceinline__ void depth_colour(const FrameConsts& fc, const FrameCounters* __restrict__ ctr,
                                             const float pw[3], float rgb[3]) {
    depth_colour_over(fc, [&] { return make_float2(ctr->depth_min, ctr->depth_max); }, pw, rgb);
}

// RasterizeMode::Normal: gaussian.wgsl:350-368, the view-space direction of the splat's third scaled axis
__device__ __forceinline__ void normal_colour(const FrameConsts& fc, const float A[3][3], const float Rm[3][3],
                                              const float sc[3], float rgb[3]) {
    float SR[3], Ln[3], wn[4];
#pragma unroll
    for (int i = 0; i < 3; ++i) SR[i] = sc[i] * Rm[i][2];
#pragma unroll
    for (int i = 0; i < 3; ++i) Ln[i] = (A[i][0] * SR[0] + A[i][1] * SR[1]) + A[i][2] * SR[2];
    mat4_dir(fc.view_from_world, Ln[0], Ln[1], Ln[2], wn);
    const float l = sqrtf(((wn[0] * wn[0] + wn[1] * wn[1]) + wn[2] * wn[2]) + wn[3] * wn[3]);
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) rgb[cc] = 0.5f * (wn[cc] / l + 1.0f);
}

// RasterizeMode::Position: gaussian.wgsl:375-376, (transformed_position - min) / (max - min)
__device__ __forceinline__ void position_colour(const FrameConsts& fc, const float pw[3], float rgb[3]) {
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) rgb[cc] = (pw[cc] - fc.aabb_min[cc]) / (fc.aabb_max[cc] - fc.aabb_min[cc]);
}

// bevy_render::maths' FRAC_PI_3 and PI_2, rounded to f32
constexpr float FRAC_PI_3_F = 1.0471975512f;
constexpr float PI_2_F = 6.28318530718f;

// bevy_render::color_operations::hsv_to_rgb: k = (vec3(5, 3, 1) + h / FRAC_PI_3) % 6.0 with WGSL's f32 remainder
// x - y * trunc(x / y), then rgb = v - v * s * max(0, min(k, min(4 - k, 1))); every step rounded, in this order
__device__ __forceinline__ void hsv_to_rgb(float h, float s, float v, float rgb[3]) {
    const float hk = h / FRAC_PI_3_F, vs = v * s;
    const float base[3] = {5.0f, 3.0f, 1.0f};
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) {
        const float x = base[cc] + hk;
        const float k = x - 6.0f * truncf(x / 6.0f);
        rgb[cc] = v - vs * fmaxf(0.0f, fminf(k, fminf(4.0f - k, 1.0f)));
    }
}

// Fixed-series atan2 in f64 (the policy replacement for WGSL atan2, optical_flow.wgsl), shared with the oracle:
// t = min(|x|, |y|) / max(|x|, |y|) in [0, 1]; above tan(pi/8), atan t = pi/4 + atan((t - 1) / (t + 1)); atan u =
// u P(u^2) by 22 odd terms (|u| <= tan(pi/8): remainder < 3e-18); then the octant and quadrant by |y| > |x| and the
// signs of x and y (IEEE atan2's values at zeros and infinities), rounded to f32.
__device__ __forceinline__ float det_atan2(float yf, float xf) {
    if (yf != yf || xf != xf) return __uint_as_float(0x7FC00000u);
    const double ay = fabs((double)yf), ax = fabs((double)xf);
    const bool steep = ay > ax;
    double t;
    if (ax == ay) t = ax == 0.0 ? 0.0 : 1.0;           // 0 / 0 and inf / inf
    else t = steep ? __ddiv_rn(ax, ay) : __ddiv_rn(ay, ax);
    double base = 0.0, u = t;
    if (t > 0.41421356237309503) { base = 0.7853981633974483; u = __ddiv_rn(__dsub_rn(t, 1.0), __dadd_rn(t, 1.0)); }
    const double z = __dmul_rn(u, u);
    double p = -1.0 / 43.0;
#pragma unroll
    for (int k = 20; k >= 0; --k) p = __dadd_rn(__dmul_rn(p, z), (k & 1 ? -1.0 : 1.0) / (double)(2 * k + 1));
    double r = __dadd_rn(base, __dmul_rn(u, p));
    if (steep) r = __dsub_rn(1.5707963267948966, r);
    if (__float_as_uint(xf) >> 31) r = __dsub_rn(3.141592653589793, r);
    if (__float_as_uint(yf) >> 31) r = -r;
    return (float)r;   // cvt.rn.f32.f64
}

// RasterizeMode::Classification (gaussian.wgsl:315-328, material/classification.wgsl:9-27): rgb holds the Color-mode
// colour (sRGB decode included); a visibility lane >= 2 mixes it half and half with the hue of class vis - 2
__device__ __forceinline__ void class_colour(const ModeConsts& mc, float vis, float rgb[3]) {
    if (vis < 2.0f) return;   // (a NaN lane takes the hue path, as in the reference)
    const float hue = ((vis - 2.0f) / (float)mc.num_classes) * 6.283185307f;
    float h[3];
    hsv_to_rgb(hue, 1.0f, 1.0f, h);
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) rgb[cc] = rgb[cc] * (1.0f - 0.5f) + h[cc] * 0.5f;   // mix(sh, hue, 0.5)
}

// RasterizeMode::OpticalFlow (gaussian.wgsl:201,369-375, material/optical_flow.wgsl:16-53): the screen motion between
// pw_prev under the previous and pw under this clip_from_world, per second, as hue = direction and saturation = speed
// (clamped to 1).  3D splats pass their transformed position as both; a 4D splat its moved and its unmoved one
__device__ __forceinline__ void flow_colour_from(const FrameConsts& fc, const ModeConsts& mc, const float pw[3],
                                                 const float pw_prev[3], float rgb[3]) {
    float c[4], cp[4];
    mat4_point(fc.clip_from_world, pw[0], pw[1], pw[2], c);
    mat4_point(mc.prev_clip_from_world, pw_prev[0], pw_prev[1], pw_prev[2], cp);
    const float mvx = (c[0] / c[3] - cp[0] / cp[3]) * 0.5f;
    const float mvy = (c[1] / c[3] - cp[1] / cp[3]) * -0.5f;
    const float fx = mvx / mc.delta_time, fy = mvy / mc.delta_time;
    const float radius = sqrtf(fx * fx + fy * fy);
    float angle = det_atan2(fy, fx);
    if (angle < 0.0f) angle = angle + PI_2_F;
    hsv_to_rgb(angle, fminf(fmaxf(radius, 0.0f), 1.0f), 1.0f, rgb);
}
__device__ __forceinline__ void flow_colour(const FrameConsts& fc, const ModeConsts& mc, const float pw[3], float rgb[3]) {
    flow_colour_from(fc, mc, pw, pw, rgb);
}

// DrawMode::HighlightSelected (gaussian.wgsl:423-427): a selected splat is drawn opaque and green in every colour source
__device__ __forceinline__ void highlight_selected(SplatRec& rec, float drgb[3], float nrgb[3]) {
    rec.r = 0.3f; rec.g = 1.0f; rec.b = 0.1f; rec.op = 1.0f;
    drgb[0] = nrgb[0] = 0.3f; drgb[1] = nrgb[1] = 1.0f; drgb[2] = nrgb[2] = 0.1f;
}

// the 48 B record, three 16 B stores
__device__ __forceinline__ void store_rec(SplatRec* __restrict__ dst, const SplatRec& rec) {
    float4* out = reinterpret_cast<float4*>(dst);
    out[0] = make_float4(rec.cx, rec.cy, rec.ux, rec.uy);
    out[1] = make_float4(rec.vx, rec.vy, __uint_as_float(rec.bx), __uint_as_float(rec.by));
    out[2] = make_float4(rec.r, rec.g, rec.b, rec.op);
}

// One entry of the index list -> the 48 B record at recs[r] (+ the 2DGS extra record and the aux colours).  An
// undrawn gaussian (outside the frustum, or unselected under DrawMode::Selected) gets an empty bbox and no colour.
// MODES2: the Classification / OpticalFlow colour sources (project_modes_kernel) instead of the four others.  SCENE (the
// scene kernels): a MODES2 segment also computes the aux colours when fc.aux is set (bgs_render_entities_aux); a
// template flag, so project_modes_kernel stays as it is.
// no_source: the frame has no colour source for this gaussian (a 3D or 2D one in a bgs_render_scene_4d Velocity frame:
// the reference builds no pipeline for it), so it stays undrawn.  Only the scene kernels pass it.
// VIEWS (project_views_aux_kernel, bgs_render_views_aux): the Depth colours are over *view_range, the segment's view's
// range, instead of the frame's.
template <bool F16, uint32_t D, bool MODES2, bool SCENE = false, bool VIEWS = false>
__device__ __forceinline__ void project_one(const FrameConsts& fc, const FrameCounters* __restrict__ ctr, uint32_t r,
                                            float4 p4, const float q[4], const float so[4], const float* sh,
                                            const float* __restrict__ cutoff_tab, uint32_t op_bits,
                                            SplatRec* __restrict__ recs, float4* __restrict__ extra,
                                            float4* __restrict__ aux, const ModeConsts& mc, bool no_source = false,
                                            const float2* __restrict__ view_range = nullptr) {
    auto depth_colour = [&](const FrameConsts& f, const FrameCounters* c, const float p[3], float rgb[3]) {
        if constexpr (VIEWS) depth_colour_over(f, [&] { return *view_range; }, p, rgb);
        else bgs::depth_colour(f, c, p, rgb);
    };
    SplatRec rec;
    rec.ux = 0.f; rec.uy = 0.f; rec.vx = 0.f; rec.vy = 0.f;
    rec.bx = BBOX_EMPTY; rec.by = BBOX_EMPTY;
    rec.r = 0.f; rec.g = 0.f; rec.b = 0.f;
    // the full model multiply, even for an identity model: keygen_world_pos's shortcut would turn a -0 into +0 here
    float pw[4], ndc[2];
    mat4_point(fc.model, p4.x, p4.y, p4.z, pw);
    const bool visible = in_frustum(fc, pw, ndc);   // gaussian.wgsl:209-210 (SORT_ALL lists hold culled gaussians too)
    const float hw = 0.5f * fc.W, hh = 0.5f * fc.H;
    rec.cx = ndc[0] * hw + hw;
    rec.cy = hh - ndc[1] * hh;
    const float opacity = so[3];
    rec.op = opacity * fc.global_opacity;
    if (visible && !no_source && !(fc.draw_mode == BGS_DRAW_SELECTED && p4.w < 0.5f)) {   // gaussian.wgsl:203-205 (DrawMode::Selected)
        const float cutoff = splat_cutoff<F16>(fc, opacity, cutoff_tab, op_bits);
        float A[3][3], Rm[3][3];   // the model 3x3 and the rotation, (row, col)
#pragma unroll
        for (int rr = 0; rr < 3; ++rr)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) A[rr][cc] = fc.model[cc * 4 + rr];
        rotation_rows(q, Rm);
        const float sc[3] = {so[0] * fc.global_scale, so[1] * fc.global_scale, so[2] * fc.global_scale};

        if (fc.gaussian_mode == BGS_GAUSSIAN_3D) {
            float c3[6];
            sigma3d(fc, A, Rm, sc, q, so, c3);
            const Cov2d v = cov2d(fc, pw, c3);
            if (fc.aabb) aabb_record(fc, v, cutoff, rec);
            else obb_record(fc, v, cutoff, rec);
        } else {
            surfel_record(fc, A, Rm, sc, pw, cutoff, r, extra, rec);
        }

        // colour source.  The Depth and Normal ones also ride along with the main one as the aux outputs
        // (bgs_render_aux, config C4): one pass yields what three single-mode frames would (the geometry and alpha of
        // a splat do not depend on the mode)
        const uint32_t mode = fc.rasterize_mode;
        float rgb[3] = {0.f, 0.f, 0.f}, drgb[3] = {0.f, 0.f, 0.f}, nrgb[3] = {0.f, 0.f, 0.f};
        if constexpr (MODES2) {
            if (mode == BGS_RASTERIZE_CLASSIFICATION) {
                sh_colour<D>(fc, A, pw, sh, rgb);
                class_colour(mc, p4.w, rgb);
            } else {
                flow_colour(fc, mc, pw, rgb);
            }
            rec.r = rgb[0]; rec.g = rgb[1]; rec.b = rgb[2];
            if constexpr (SCENE) {
                if (fc.aux) {
                    depth_colour(fc, ctr, pw, drgb);
                    normal_colour(fc, A, Rm, sc, nrgb);
                }
            }
        } else {
            if (mode == BGS_RASTERIZE_COLOR) sh_colour<D>(fc, A, pw, sh, rgb);
            if (mode == BGS_RASTERIZE_POSITION) position_colour(fc, pw, rgb);
            if (mode == BGS_RASTERIZE_DEPTH || fc.aux) depth_colour(fc, ctr, pw, drgb);
            if (mode == BGS_RASTERIZE_NORMAL || fc.aux) normal_colour(fc, A, Rm, sc, nrgb);
            const bool depth = mode == BGS_RASTERIZE_DEPTH, normal = mode == BGS_RASTERIZE_NORMAL;
            rec.r = depth ? drgb[0] : normal ? nrgb[0] : rgb[0];
            rec.g = depth ? drgb[1] : normal ? nrgb[1] : rgb[1];
            rec.b = depth ? drgb[2] : normal ? nrgb[2] : rgb[2];
        }
        if (fc.draw_mode == BGS_DRAW_HIGHLIGHT_SELECTED && p4.w > 0.5f) highlight_selected(rec, drgb, nrgb);
        if (fc.aux && aux != nullptr) {
            aux[(size_t)r * 2] = make_float4(drgb[0], drgb[1], drgb[2], 0.0f);
            aux[(size_t)r * 2 + 1] = make_float4(nrgb[0], nrgb[1], nrgb[2], 0.0f);
        }
    }
    store_rec(recs + r, rec);
}

// 128 threads at up to 128 registers (no spills).  Beside the depth sort an SM has shared memory for one such CTA, so
// a tighter register bound buys no occupancy there, and with several frames in flight fewer, fatter CTAs measured
// faster than 6 or 8 per SM (DESIGN.md section 9).
constexpr int PROJ_THREADS = 128, PROJ_WARPS = PROJ_THREADS / 32, PROJ_MIN_CTAS = 4;

// The projection loop of every projection kernel.  Record r of n_vis is entry r of the source's list (entry_src.cuh):
//   one cloud, by_slot: r is a compact slot (ascending gaussian index; runs concurrently with the depth sort)
//   one cloud, else   : r is a front-to-back rank, the list is the far->near sorted index list
//   a scene           : r is a compact slot, its entry a global index; the launch projects the entries whose segment
//                       Src::mine covers, each with its segment's constants
// The grid is persistent and each warp strides over groups of 32 entries with two groups in flight: once the lanes
// hold group i's attributes in registers, the copies of group i + 1 start filling the warp's stage and the list
// entries of group i + 2 are on their way into a register, so both dependent memory latencies sit under project_one.
// Geo is the splat geometry: chunks per entry in the stage (SCH) and in the block (BCH), the pieces copied when the
// colour source does not read the SH coefficients (GEO), read (an entry's position, q, so and EXT more floats out of
// the stage) and project (its record).  The registers are plain arrays of this loop: gathered into a struct, they
// change how ptxas allocates the benchmarked project_kernel.
template <class Src, class Geo>
__device__ __forceinline__ void project_loop(const Src& src, const Geo& geo, const FrameCounters* __restrict__ ctr,
                                             const ModeConsts& mc) {
    __shared__ __align__(16) uint4 s_stages[PROJ_WARPS][32 * Geo::SCH];   // 3D degree 3: f16 16 KB, f32 32 KB; 4D 16 KB
    const int lane = threadIdx.x & 31;
    uint4* const stage = s_stages[threadIdx.x >> 5];
    const uint32_t n_vis = ctr->n_vis, stride = gridDim.x * PROJ_THREADS;
    auto gather = [&](uint32_t r0, uint32_t e) {   // one commit group per call, empty past the list's end
        const uint32_t n_valid = r0 < n_vis ? n_vis - r0 : 0u;
        if (geo.need_sh) src.template copy<Geo::SCH, Geo::SCH, Geo::BCH>(e, n_valid, stage, lane);
        else src.template copy<Geo::SCH, Geo::GEO, Geo::BCH>(e, n_valid, stage, lane);
        cp_async_commit();
    };
    uint32_t r0 = (blockIdx.x * PROJ_WARPS + (threadIdx.x >> 5)) * 32u;
    uint32_t e = src.entry(r0 + lane, n_vis);
    gather(r0, e);
    uint32_t e_next = src.entry(r0 + stride + lane, n_vis);
    for (; r0 < n_vis; r0 += stride) {
        cp_async_wait<0>();
        __syncwarp();   // every lane's copies of this group have landed
        const uint32_t r = r0 + lane, j = src.seg(e);
        const bool mine = r < n_vis && (!Src::SEGMENTED || src.mine(j));
        float ext[Geo::EXT], q[4], so[4];
        uint32_t op_bits = 0u;
        float4 p4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (mine) p4 = geo.read(stage, lane, ext, q, so, op_bits);
        __syncwarp();   // the stage is read out before the next group's copies overwrite it
        const uint32_t e_mine = e;
        gather(r0 + stride, e_next);
        e = e_next;
        e_next = src.entry(r0 + 2u * stride + lane, n_vis);
        if (mine) geo.project(src, j, e_mine, r, p4, q, so, ext, op_bits, mc);
    }
}

// The 3D and 2D splats: Attr<F16, D>'s blocks and project_one's record.  MODES2: project_modes_kernel's colour sources.
// VIEWS: segment j's Depth colours are over view_range[j / k] (project_views_aux_kernel).
template <bool F16, uint32_t D, bool MODES2, bool VIEWS = false>
struct Geo3d {
    using A = Attr<F16, D>;
    static constexpr int SCH = A::CH, BCH = A::CH, GEO = A::GEO, EXT = sh_floats(D);
    const FrameCounters* ctr;
    bool need_sh;   // the colour source reads the SH coefficients
    SplatRec* recs;
    float4* extra;
    const float* cutoff_tab;
    float4* aux;
    const float2* view_range = nullptr;
    uint32_t k = 0u;   // segments per view

    __device__ __forceinline__ float4 read(const uint4* stage, int lane, float* sh, float q[4], float so[4], uint32_t& op_bits) const {
        return A::load(stage, lane, sh, q, so, need_sh, op_bits);
    }
    template <class Src>
    __device__ __forceinline__ void project(const Src& src, uint32_t j, uint32_t, uint32_t r, float4 p4, const float q[4],
                                            const float so[4], const float* sh, uint32_t op_bits, const ModeConsts& mc) const {
        const FrameConsts& fc = src.fc(j);
        project_one<F16, D, MODES2, Src::SEGMENTED, VIEWS>(fc, ctr, r, p4, q, so, sh, cutoff_tab, op_bits, recs, extra, aux, mc,
                                                           MODES2 && Src::SEGMENTED && fc.rasterize_mode == BGS_RASTERIZE_VELOCITY,
                                                           VIEWS ? view_range + j / k : nullptr);
    }
};

template <bool F16, uint32_t D>
__global__ void __launch_bounds__(PROJ_THREADS, PROJ_MIN_CTAS)
project_kernel(const void* __restrict__ blocks, const uint32_t* __restrict__ index_list, int by_slot,
               const FrameCounters* __restrict__ ctr, FrameConsts fc, SplatRec* __restrict__ recs,
               float4* __restrict__ extra /* 4 x float4 per record, 2DGS + USE_AABB only */, const float* __restrict__ cutoff_tab,
               float4* __restrict__ aux /* 2 x float4 per record (depth rgb, normal rgb), bgs_render_aux only */) {
    project_loop(OneCloud{nullptr, fc, static_cast<const uint4*>(blocks), index_list, by_slot},
                 Geo3d<F16, D, false>{ctr, fc.rasterize_mode == BGS_RASTERIZE_COLOR, recs, extra, cutoff_tab, aux},
                 ctr, ModeConsts{});
}

// project_kernel for RasterizeMode::Classification / OpticalFlow (bgs_render_ex): the same records but for r, g, b.  A
// kernel of its own, so that project_kernel's mode branch (and its register budget) stays as it is.
template <bool F16, uint32_t D>
__global__ void __launch_bounds__(PROJ_THREADS, PROJ_MIN_CTAS)
project_modes_kernel(const void* __restrict__ blocks, const uint32_t* __restrict__ index_list, int by_slot,
                     const FrameCounters* __restrict__ ctr, FrameConsts fc, ModeConsts mc, SplatRec* __restrict__ recs,
                     float4* __restrict__ extra, const float* __restrict__ cutoff_tab) {
    // OpticalFlow reads the position only
    project_loop(OneCloud{nullptr, fc, static_cast<const uint4*>(blocks), index_list, by_slot},
                 Geo3d<F16, D, true>{ctr, fc.rasterize_mode == BGS_RASTERIZE_CLASSIFICATION, recs, extra, cutoff_tab, nullptr},
                 ctr, mc);
}

// ---- scene frames (the segment table, common.cuh): the depth range, and the projection group of a cloud's segments
void launch_depth_range_scene(const SceneTable& tab, const uint32_t* sorted_payload, const uint32_t* slot_ids, FrameCounters* ctr,
                              cudaStream_t stream) {
    depth_range_scene_kernel<<<1, 32, 0, stream>>>(tab, sorted_payload, slot_ids, ctr);
}

uint32_t project_group(CloudLayout layout, uint32_t sh_degree) {
    if (is_4d(layout)) return PROJECT_GROUP_4D;   // (launch_project_4d_scene)
    return (is_f16(layout) ? 1u : 0u) | sh_degree << 1;
}

// ---- Gaussian4d (bgs_render_4d; the rule is include/bgs.h's).  Matrices [col][row], as WGSL indexes them.

// gaussian_4d.wgsl:37-130: Sigma of the 4D gaussian conditioned on time t
struct Cond4d {
    float c3[6];       // the conditioned 3D covariance, WGSL [0][0], [0][1], [0][2], [1][1], [1][2], [2][2]
    float dm[3];       // delta_mean
    float marginal;    // marginal_t
    bool mask;         // marginal_t > 0.05 (false for NaN)
};
__device__ __forceinline__ Cond4d condition_4d(float gs, const float ql[4], const float qr[4], const float so[4], float timestamp,
                                               float timescale, float t) {
    Cond4d g;
    const float dt = t - timestamp;
    const float sd[4] = {gs * so[0], gs * so[1], gs * so[2], timescale};
    const float w = ql[0], x = ql[1], y = ql[2], z = ql[3];
    const float wr = qr[0], xr = qr[1], yr = qr[2], zr = qr[3];
    const float Ml[4][4] = {{w, -x, -y, -z}, {x, w, -z, y}, {y, z, w, -x}, {z, -y, x, w}};
    const float Mr[4][4] = {{wr, -xr, -yr, -zr}, {xr, wr, zr, -yr}, {yr, -zr, wr, xr}, {zr, yr, -xr, wr}};
    float M[4][4];   // M = (M_r * M_l) * S: R[c][r] = sum_k M_r[k][r] M_l[c][k], then column c times S[c][c]
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r)
            M[c][r] = (((Mr[0][r] * Ml[c][0] + Mr[1][r] * Ml[c][1]) + Mr[2][r] * Ml[c][2]) + Mr[3][r] * Ml[c][3]) * sd[c];
    // Sigma = transpose(M) * M: Sigma[c][r] = sum_k M[r][k] M[c][k]
    auto sig = [&](int c, int r) {
        return ((M[r][0] * M[c][0] + M[r][1] * M[c][1]) + M[r][2] * M[c][2]) + M[r][3] * M[c][3];
    };
    const float cov_t = sig(3, 3);
    g.marginal = det_exp(((-0.5f * dt) * dt) / cov_t);
    g.mask = g.marginal > 0.05f;
#pragma unroll
    for (int i = 0; i < 6; ++i) g.c3[i] = 0.0f;
    g.dm[0] = g.dm[1] = g.dm[2] = 0.0f;
    if (!g.mask) return g;
    const float c12[3] = {sig(0, 3), sig(1, 3), sig(2, 3)};
    auto cond = [&](int c, int r) { return sig(c, r) - (c12[c] * c12[r]) / cov_t; };
    g.c3[0] = cond(0, 0); g.c3[1] = cond(0, 1); g.c3[2] = cond(0, 2);
    g.c3[3] = cond(1, 1); g.c3[4] = cond(1, 2); g.c3[5] = cond(2, 2);
#pragma unroll
    for (int i = 0; i < 3; ++i) g.dm[i] = (c12[i] / cov_t) * dt;
    return g;
}

// spherindrical_harmonics.wgsl:11-126: the SH-3 colour plus cos(2 pi theta) and cos(4 pi theta) times the second and
// third 48 coefficients, theta = dt / duration.  The coefficients stream from the block (gaussian-major, 36 chunks from
// sh) a chunk at a time: only drawn splats of the colour sources that read them ever fetch them.
constexpr float PI_F = 3.14159274f;   // radians(180.0) in f32
__device__ __forceinline__ void spherindrical_colour(const FrameConsts& fc, const TemporalConsts& tc, const float A[3][3],
                                                     const float pw[3], float dt, const uint4* __restrict__ sh, float rgb[3]) {
    float basis[16];
    sh_basis(fc, A, pw, basis);
    float acc[3][3];   // [section][channel]: the SH-3 colour (from 0.5), then the two time sums (from 0)
#pragma unroll
    for (int t = 0; t < 3; ++t) { acc[t][0] = t ? 0.0f : 0.5f; acc[t][1] = acc[t][0]; acc[t][2] = acc[t][0]; }
#pragma unroll
    for (int q = 0; q < 36; ++q) {
        const uint4 v = __ldg(sh + q);
        const float f[4] = {__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w)};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int j = 4 * q + e, t = j / 48, k = (j % 48) / 3, cc = j % 3;
            acc[t][cc] = fmaf(f[e], basis[k], acc[t][cc]);   // colour: FMA is fine
        }
    }
    const float theta = dt / tc.duration;
    const float t1 = det_cos((2.0f * PI_F) * theta), t2 = det_cos((4.0f * PI_F) * theta);
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) {
        rgb[cc] = (acc[0][cc] + t1 * acc[1][cc]) + t2 * acc[2][cc];
        if (fc.color_space == 0u) rgb[cc] = srgb_to_linear(rgb[cc]);
    }
}

// RasterizeMode::Velocity (gaussian.wgsl:378-405): the splat's velocity in the local frame by a forward difference of
// 1e-3; opacity 0 (and rgb 0: the reference's NaN) below 1 % of the magnitude scale
__device__ __forceinline__ void velocity_colour(const Cond4d& now, const Cond4d& fut, float rgb[3], float& opacity) {
    float v[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) v[i] = ((fut.mask ? fut.dm[i] : 0.0f) - now.dm[i]) / 1.0e-3f;
    const float len = sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    const float scaled = fminf(fmaxf((len - 1.0f) / (2.0f - 1.0f), 0.0f), 1.0f);
    if (scaled < 1.0e-2f) {
        opacity = 0.0f;
        rgb[0] = rgb[1] = rgb[2] = 0.0f;
        return;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) rgb[i] = (0.5f * (v[i] / len + 1.0f)) * scaled;
}

// One entry of the index list of a 4D cloud -> its record at recs[r] (and, on depth-tested frames, its splat depth).
// Undrawn (outside the frustum at the base position, unselected under DrawMode::Selected, masked by time, or outside
// the frustum at the moved position): the base position's centre, the stored opacity, an empty bbox and no colour.
__device__ __forceinline__ void project_one_4d(const FrameConsts& fc, const ModeConsts& mc, const TemporalConsts& tc,
                                               const FrameCounters* __restrict__ ctr, uint32_t r, float4 p4, const float ql[4],
                                               const float qr[4], const float so[4], const float tt[4],
                                               const uint4* __restrict__ sh, SplatRec* __restrict__ recs,
                                               float* __restrict__ depths) {
    SplatRec rec;
    rec.ux = 0.f; rec.uy = 0.f; rec.vx = 0.f; rec.vy = 0.f;
    rec.bx = BBOX_EMPTY; rec.by = BBOX_EMPTY;
    rec.r = 0.f; rec.g = 0.f; rec.b = 0.f;
    float pw[4], ndc[2];
    mat4_point(fc.model, p4.x, p4.y, p4.z, pw);
    const bool visible = in_frustum(fc, pw, ndc);   // every depth width culls on the base position (include/bgs.h)
    const float hw = 0.5f * fc.W, hh = 0.5f * fc.H;
    rec.cx = ndc[0] * hw + hw;
    rec.cy = hh - ndc[1] * hh;
    const float opacity = so[3];
    rec.op = opacity * fc.global_opacity;
    float pm[4] = {pw[0], pw[1], pw[2], pw[3]};   // the position the record's centre comes from
    if (visible && !(fc.draw_mode == BGS_DRAW_SELECTED && p4.w < 0.5f)) {
        const float cutoff = splat_cutoff<false>(fc, opacity, nullptr, 0u);   // from the stored opacity
        const Cond4d g = condition_4d(fc.global_scale, ql, qr, so, tt[0], tt[1], tc.time);
        float nm[2];
        if (g.mask) mat4_point(fc.model, p4.x + g.dm[0], p4.y + g.dm[1], p4.z + g.dm[2], pm);
        if (g.mask && in_frustum(fc, pm, nm)) {
            rec.cx = nm[0] * hw + hw;
            rec.cy = hh - nm[1] * hh;
            float op = opacity * g.marginal;
            const Cov2d v = cov2d(fc, pm, g.c3);   // (the model 3x3 does not touch cov3d)
            if (fc.aabb) aabb_record(fc, v, cutoff, rec);
            else obb_record(fc, v, cutoff, rec);
            float A[3][3];
#pragma unroll
            for (int rr = 0; rr < 3; ++rr)
#pragma unroll
                for (int cc = 0; cc < 3; ++cc) A[rr][cc] = fc.model[cc * 4 + rr];
            const uint32_t mode = fc.rasterize_mode;
            float rgb[3] = {0.f, 0.f, 0.f};
            if (mode == BGS_RASTERIZE_COLOR || mode == BGS_RASTERIZE_CLASSIFICATION) {
                spherindrical_colour(fc, tc, A, pm, tc.time - tt[0], sh, rgb);
                if (mode == BGS_RASTERIZE_CLASSIFICATION) class_colour(mc, p4.w, rgb);
            } else if (mode == BGS_RASTERIZE_DEPTH) {
                depth_colour(fc, ctr, pm, rgb);
            } else if (mode == BGS_RASTERIZE_POSITION) {
                position_colour(fc, pm, rgb);
            } else if (mode == BGS_RASTERIZE_OPTICAL_FLOW) {
                flow_colour_from(fc, mc, pm, pw, rgb);   // the previous position is the unmoved one (gaussian.wgsl:201)
            } else {
                const Cond4d fut = condition_4d(fc.global_scale, ql, qr, so, tt[0], tt[1], tc.time_future);
                velocity_colour(g, fut, rgb, op);
            }
            rec.r = rgb[0]; rec.g = rgb[1]; rec.b = rgb[2];
            rec.op = op * fc.global_opacity;
            float unused[3];
            if (fc.draw_mode == BGS_DRAW_HIGHLIGHT_SELECTED && p4.w > 0.5f) highlight_selected(rec, unused, unused);
        } else {
            pm[0] = pw[0]; pm[1] = pw[1]; pm[2] = pw[2];
        }
    }
    store_rec(recs + r, rec);
    if (depths) depths[r] = splat_depth(fc, pm);
}

// The 4D block is 768 B: a warp stages only each entry's first 128 B line (position, both rotations, scale-opacity,
// timestamp-timescale; 4 KB per warp), piece p of entry g at g * GEO4 + stage_slot<GEO4>(p, g).  The coefficients stay
// in global memory until a drawn splat's colour needs them.
constexpr int CH4 = (int)chunks(CloudLayout::F32x4D, SH_DEGREE_MAX), GEO4 = 8;
struct Geo4d {
    static constexpr int SCH = GEO4, BCH = CH4, GEO = GEO4, EXT = 8;
    static constexpr bool need_sh = false;
    const FrameCounters* ctr;
    SplatRec* recs;
    float* depths;   // depth-tested frames only

    // q: rotation, so: scale-opacity, ext: rotation_r, then timestamp-timescale
    __device__ __forceinline__ float4 read(const uint4* stage, int lane, float ext[8], float q[4], float so[4], uint32_t&) const {
        auto piece = [&](int p, float* out) {
            const uint4 v = stage[lane * GEO4 + stage_slot<GEO4>(p, lane)];
            out[0] = __uint_as_float(v.x); out[1] = __uint_as_float(v.y); out[2] = __uint_as_float(v.z); out[3] = __uint_as_float(v.w);
        };
        float p4[4];
        piece(POS_CHUNK, p4); piece(SECOND_CHUNK, q); piece(ROT_R_CHUNK, ext); piece(SO_4D_CHUNK, so); piece(TT_CHUNK, ext + 4);
        return make_float4(p4[0], p4[1], p4[2], p4[3]);
    }
    template <class Src>
    __device__ __forceinline__ void project(const Src& src, uint32_t j, uint32_t e, uint32_t r, float4 p4, const float q[4],
                                            const float so[4], const float ext[8], uint32_t, const ModeConsts& mc) const {
        project_one_4d(src.fc(j), mc, src.tc(j), ctr, r, p4, q, ext, so, ext + 4,
                       src.template block_at<CH4>(j, e) + sh_first(CloudLayout::F32x4D), recs, depths);
    }
};

__global__ void __launch_bounds__(PROJ_THREADS, PROJ_MIN_CTAS)
project_4d_kernel(const uint4* __restrict__ blocks, const uint32_t* __restrict__ index_list, int by_slot,
                  const FrameCounters* __restrict__ ctr, FrameConsts fc, ModeConsts mc, TemporalConsts tc,
                  SplatRec* __restrict__ recs, float* __restrict__ depths /* depth-tested frames only */) {
    project_loop(OneCloud{nullptr, fc, blocks, index_list, by_slot, &tc}, Geo4d{ctr, recs, depths}, ctr, mc);
}

void launch_project_4d(const void* blocks, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                       const FrameConsts& fc, const ModeConsts& mc, const TemporalConsts& tc, SplatRec* recs, float* depths,
                       uint32_t n_hint, int sm_count, cudaStream_t stream) {
    const uint32_t grid = persistent_grid(n_hint, PROJ_THREADS, PROJ_MIN_CTAS, sm_count);
    project_4d_kernel<<<grid, PROJ_THREADS, 0, stream>>>(static_cast<const uint4*>(blocks), index_list, by_slot, ctr, fc, mc, tc,
                                                         recs, depths);
}

// ---- Scene frames (bgs_render_scene, _scene_4d and _entities): the projection over a segment table (common.cuh).
// Record r is compact slot r, whose global index slot_ids[r] lies in segment j: its block is gaussian slot_ids[r] -
// offset of cloud j's blocks, and project_one / project_one_4d run with segment j's FrameConsts (its entity's settings),
// times and num_classes, so the record is the one a frame of cloud j alone would write.  One launch per group
// (project_group, | ENTITY_MODES for the Classification / OpticalFlow / Velocity kernel, or PROJECT_GROUP_4D): its warps
// stride over every slot and project those whose segment is in the group; need_sh says whether one of the group's
// segments reads the SH coefficients.

// (the f32 blocks of degree 2 and 3 hold 48 SH floats in registers beside the segment's constants: 3 CTAs per SM keeps
// them from spilling)
template <bool F16, uint32_t D>
constexpr int scene_min_ctas() { return !F16 && D >= 2 ? 3 : PROJ_MIN_CTAS; }

// G's projection with segment j's num_classes (classes.n[j]: a SceneClasses, or a SceneTableDev's array)
struct ClassesDev {
    const uint32_t* n;
};
template <class G, class Classes = SceneClasses>
struct SceneGeo : G {
    const Classes& classes;
    template <class Src>
    __device__ __forceinline__ void project(const Src& src, uint32_t j, uint32_t e, uint32_t r, float4 p4, const float q[4],
                                            const float so[4], const float* ext, uint32_t op_bits, const ModeConsts& mc) const {
        ModeConsts m = mc;
        m.num_classes = classes.n[j];
        G::project(src, j, e, r, p4, q, so, ext, op_bits, m);
    }
};

template <bool F16, uint32_t D, bool MODES2>
__global__ void __launch_bounds__(PROJ_THREADS, scene_min_ctas<F16, D>())
project_scene_kernel(SceneTable tab, uint32_t group, uint32_t need_sh, SceneClasses classes, ModeConsts mc,
                     const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr, SplatRec* __restrict__ recs,
                     float4* __restrict__ extra, const float* __restrict__ cutoff_tab,
                     float4* __restrict__ aux /* bgs_render_entities_aux only */) {
    project_loop(SceneSrc{tab, 1u << group, slot_ids},
                 SceneGeo<Geo3d<F16, D, MODES2>>{{ctr, need_sh != 0u, recs, extra, cutoff_tab, aux}, classes}, ctr, mc);
}

// bgs_render_views_aux's projection: project_scene_kernel's, with each segment's Depth colours (its colour source and its
// aux depth colour) over its view's range, vr->range[j / k].  A kernel of its own, so the other scene frames keep
// project_scene_kernel as it is.
template <bool F16, uint32_t D, bool MODES2>
__global__ void __launch_bounds__(PROJ_THREADS, scene_min_ctas<F16, D>())
project_views_aux_kernel(SceneTable tab, uint32_t group, uint32_t need_sh, SceneClasses classes, ModeConsts mc,
                         const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                         SplatRec* __restrict__ recs, float4* __restrict__ extra, const float* __restrict__ cutoff_tab,
                         float4* __restrict__ aux, const ViewRanges* __restrict__ vr, uint32_t k) {
    project_loop(SceneSrc{tab, 1u << group, slot_ids},
                 SceneGeo<Geo3d<F16, D, MODES2, true>>{{ctr, need_sh != 0u, recs, extra, cutoff_tab, aux, vr->range, k}, classes},
                 ctr, mc);
}

// ---- bgs_render_views_aux: each view's Depth range (ViewRanges) from one pass over the n_vis sorted visible entries.
// The joint sort is stable and view i's global indices are [i n, (i + 1) n), so view i's entries keep, in the joint
// sorted list, the order of its own frame's sort.  Its list's sorted[1] is then its second visible entry (with fewer than
// two visible: its first culled index), and its sorted[n - 1] its last culled index (with none culled: its last visible
// entry).  The culled ends come from slot_ids: the stable compaction keeps a view's visible global indices as one
// ascending run, so its first culled index is where that run first departs from i n, i n + 1, ..., and its last culled
// index where the run, read backwards, first departs from (i + 1) n - 1, (i + 1) n - 2, ...
constexpr int DRV_THREADS = 256, DRV_CTAS_PER_SM = 4;

// sorted position p into a ViewRanges::first2 word (shared or global): kept when it is among the two smallest so far
__device__ __forceinline__ void first2_insert(unsigned long long* w, uint32_t p) {
    const unsigned long long x = 0xFFFFFFFFu - p;
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(w);
    for (;;) {
        const unsigned long long a = cur >> 32, b = cur & 0xFFFFFFFFull;
        unsigned long long next;
        if (x > a) next = x << 32 | a;
        else if (x > b) next = a << 32 | x;
        else return;
        const unsigned long long prev = atomicCAS(w, cur, next);
        if (prev == cur) return;
        cur = prev;
    }
}

// the smallest t in [0, len) with miss(t), len if none, for a miss() that stays true once true: a 32-way search, the
// whole warp calling it (miss is read only below len)
template <class Miss>
__device__ __forceinline__ uint32_t warp_first_miss(uint32_t len, Miss miss) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t lo = 0u, hi = len;   // the answer lies in [lo, hi]
    while (lo < hi) {
        const uint32_t step = (hi - lo + 31u) / 32u, t = lo + lane * step;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, t >= hi || miss(t));
        if (m == 0u) {
            lo += 31u * step + 1u;
        } else {
            const uint32_t f = (uint32_t)__ffs(m) - 1u;
            hi = min(hi, lo + f * step);
            if (f > 0u) lo += (f - 1u) * step + 1u;
        }
    }
    return lo;
}

__global__ void __launch_bounds__(DRV_THREADS)
depth_range_views_kernel(SceneTable tab, uint32_t v, uint32_t n_view, const uint32_t* __restrict__ sorted_payload,
                         const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                         ViewRanges* __restrict__ vr) {
    __shared__ unsigned long long s_first2[MAX_VIEWS];
    __shared__ uint32_t s_last_p1[MAX_VIEWS], s_cnt[MAX_VIEWS];
    __shared__ bool s_final;
    const uint32_t t = threadIdx.x, lane = t & 31u;
    if (t < MAX_VIEWS) { s_first2[t] = 0ull; s_last_p1[t] = 0u; s_cnt[t] = 0u; }
    __syncthreads();
    // the pass: each warp's lanes hold consecutive positions, so a view's lowest two lanes in the warp are its warp's
    // first two positions and its highest lane its last
    const uint32_t n_vis = ctr->n_vis;
    for (uint32_t p0 = blockIdx.x * DRV_THREADS; p0 < n_vis; p0 += gridDim.x * DRV_THREADS) {
        const uint32_t p = p0 + t;
        const uint32_t view = p < n_vis ? __ldg(slot_ids + __ldg(sorted_payload + p)) / n_view : 0xFFFFFFFFu;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, view);
        if (view != 0xFFFFFFFFu) {
            const uint32_t rank = __popc(peers & lanemask_lt());
            if (rank == 0u) atomicAdd(&s_cnt[view], (uint32_t)__popc(peers));
            if (rank < 2u) first2_insert(&s_first2[view], p);
            if ((peers >> lane) == 1u) atomicMax(&s_last_p1[view], p + 1u);
        }
    }
    __syncthreads();
    if (t < v) {
        const unsigned long long f = s_first2[t];
        if (f >> 32) first2_insert(&vr->first2[t], 0xFFFFFFFFu - (uint32_t)(f >> 32));
        if (f & 0xFFFFFFFFull) first2_insert(&vr->first2[t], 0xFFFFFFFFu - (uint32_t)f);
        if (s_last_p1[t]) atomicMax(&vr->last_p1[t], s_last_p1[t]);
        if (s_cnt[t]) atomicAdd(&vr->n_vis[t], s_cnt[t]);
    }
    __threadfence();
    __syncthreads();
    if (t == 0) s_final = atomicAdd(&vr->done, 1u) == gridDim.x - 1u;
    __syncthreads();
    // the last CTA past the pass: every view's range, one warp per view
    if (!s_final || n_view < 2u) return;   // (n < 2: the range stays (0, 0) and depth_colour draws black, as one view's)
    __threadfence();
    const volatile ViewRanges* w = vr;
    const SceneSrc src{tab};
    auto dist = [&](uint32_t id) {   // depth_range_body's
        const uint32_t j = src.seg(id);
        const FrameConsts& fc = src.fc(j);
        const float4 p = *src.pos_at(j, id);
        float pw[4];
        mat4_point(fc.model, p.x, p.y, p.z, pw);
        return sqrtf(cam_dist2(fc, pw));
    };
    auto id_at = [&](uint32_t pos) { return __ldg(slot_ids + __ldg(sorted_payload + pos)); };
    for (uint32_t i = t >> 5; i < v; i += DRV_THREADS / 32) {
        const uint32_t cnt = w->n_vis[i], last_p1 = w->last_p1[i];
        const unsigned long long f = w->first2[i];
        uint32_t run0 = 0u;   // the view's first compact slot
        for (uint32_t e = 0; e < i; ++e) run0 += w->n_vis[e];
        const uint32_t base = i * n_view;
        const uint32_t lo = warp_first_miss(cnt, [&](uint32_t x) { return __ldg(slot_ids + run0 + x) != base + x; });
        const uint32_t hi = warp_first_miss(cnt, [&](uint32_t x) {
            return __ldg(slot_ids + run0 + cnt - 1u - x) != base + n_view - 1u - x;
        });
        const uint32_t first = cnt >= 2u ? id_at(0xFFFFFFFFu - (uint32_t)(f & 0xFFFFFFFFull)) : base + lo;
        const uint32_t last = cnt < n_view ? base + n_view - 1u - hi : id_at(last_p1 - 1u);
        if (lane == 0u) vr->range[i] = make_float2(dist(last), dist(first));
    }
}

__global__ void __launch_bounds__(PROJ_THREADS, PROJ_MIN_CTAS)
project_4d_scene_kernel(SceneTable tab, SceneTimes times, SceneClasses classes, ModeConsts mc,
                        const uint32_t* __restrict__ slot_ids, const FrameCounters* __restrict__ ctr,
                        SplatRec* __restrict__ recs, float* __restrict__ depths /* depth-tested frames only */) {
    project_loop(SceneSrc{tab, 1u << PROJECT_GROUP_4D, slot_ids, times.t}, SceneGeo<Geo4d>{{ctr, recs, depths}, classes}, ctr, mc);
}
// sm_90 takes up to 32764 B of kernel parameters (CUDA >= 12.1): the table (~22 KB), the times (768 B), the classes
// (256 B), the extras and four pointers
static_assert(sizeof(SceneTable) + sizeof(SceneTimes) + sizeof(SceneClasses) + sizeof(ModeConsts) + 4 * sizeof(void*) + 16 <= 32764,
              "project_4d_scene_kernel's parameters exceed the sm_90 limit");
// (project_views_aux_kernel: the table, the classes, the extras, seven pointers and three words)
static_assert(sizeof(SceneTable) + sizeof(SceneClasses) + sizeof(ModeConsts) + 7 * sizeof(void*) + 16 <= 32764,
              "project_views_aux_kernel's parameters exceed the sm_90 limit");

void launch_project_scene(const SceneTable& tab, uint32_t group, bool need_sh, const SceneClasses& classes,
                          const ModeConsts& mc, const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs,
                          float4* extra, uint32_t n_hint, int sm_count, const float* cutoff_tab, float4* aux,
                          cudaStream_t stream, const ViewRanges* view_ranges, uint32_t k) {
    const uint32_t grid = persistent_grid(n_hint, PROJ_THREADS, PROJ_MIN_CTAS, sm_count);
    const uint32_t g = group & ~ENTITY_MODES;
    with_layout_degree(g & 1u ? CloudLayout::F16 : CloudLayout::F32, g >> 1, [&](auto L, auto Dt) {
        constexpr CloudLayout Lv = decltype(L)::value;
        constexpr uint32_t D = decltype(Dt)::value;
        if constexpr (!is_4d(Lv)) {
            if (view_ranges) {
                auto* kernel = (group & ENTITY_MODES) ? project_views_aux_kernel<is_f16(Lv), D, true>
                                                      : project_views_aux_kernel<is_f16(Lv), D, false>;
                kernel<<<grid, PROJ_THREADS, 0, stream>>>(tab, group, need_sh ? 1u : 0u, classes, mc, slot_ids, ctr, recs, extra,
                                                          cutoff_tab, aux, view_ranges, k);
                return;
            }
            auto* kernel = (group & ENTITY_MODES) ? project_scene_kernel<is_f16(Lv), D, true>
                                                  : project_scene_kernel<is_f16(Lv), D, false>;
            kernel<<<grid, PROJ_THREADS, 0, stream>>>(tab, group, need_sh ? 1u : 0u, classes, mc, slot_ids, ctr, recs, extra,
                                                      cutoff_tab, aux);
        }
    });
}

// ---- bgs_render_entities_many: the scene kernels over a segment table in device memory (SceneSrcDev), their bodies
// the scene frames' own
__global__ void depth_range_many_kernel(SceneTableDev tab, const uint32_t* __restrict__ sorted_payload,
                                        const uint32_t* __restrict__ slot_ids, FrameCounters* __restrict__ ctr) {
    depth_range_body(SceneSrcDev{tab}, tab.n_total, sorted_payload, slot_ids, ctr);
}

template <bool F16, uint32_t D, bool MODES2>
__global__ void __launch_bounds__(PROJ_THREADS, scene_min_ctas<F16, D>())
project_many_kernel(SceneTableDev tab, uint32_t group, uint32_t need_sh, ModeConsts mc, const uint32_t* __restrict__ slot_ids,
                    const FrameCounters* __restrict__ ctr, SplatRec* __restrict__ recs, float4* __restrict__ extra,
                    const float* __restrict__ cutoff_tab) {
    project_loop(SceneSrcDev{tab, 1u << group, slot_ids},
                 SceneGeo<Geo3d<F16, D, MODES2>, ClassesDev>{{ctr, need_sh != 0u, recs, extra, cutoff_tab, nullptr},
                                                             ClassesDev{tab.classes}},
                 ctr, mc);
}

// (the segment's constants come from global memory: at PROJ_MIN_CTAS per SM its 128 registers spill 4 B; at 3, 168
// registers and no spill)
constexpr int PROJ_4D_MANY_CTAS = 3;
__global__ void __launch_bounds__(PROJ_THREADS, PROJ_4D_MANY_CTAS)
project_4d_many_kernel(SceneTableDev tab, ModeConsts mc, const uint32_t* __restrict__ slot_ids,
                       const FrameCounters* __restrict__ ctr, SplatRec* __restrict__ recs, float* __restrict__ depths) {
    project_loop(SceneSrcDev{tab, 1u << PROJECT_GROUP_4D, slot_ids, tab.times},
                 SceneGeo<Geo4d, ClassesDev>{{ctr, recs, depths}, ClassesDev{tab.classes}}, ctr, mc);
}

void launch_depth_range_many(const SceneTableDev& tab, const uint32_t* sorted_payload, const uint32_t* slot_ids,
                             FrameCounters* ctr, cudaStream_t stream) {
    depth_range_many_kernel<<<1, 32, 0, stream>>>(tab, sorted_payload, slot_ids, ctr);
}

void launch_project_many(const SceneTableDev& tab, uint32_t group, bool need_sh, const ModeConsts& mc,
                         const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs, float4* extra,
                         float* depths, uint32_t n_hint, int sm_count, const float* cutoff_tab, cudaStream_t stream) {
    if (group == PROJECT_GROUP_4D) {
        const uint32_t grid = persistent_grid(n_hint, PROJ_THREADS, PROJ_4D_MANY_CTAS, sm_count);
        project_4d_many_kernel<<<grid, PROJ_THREADS, 0, stream>>>(tab, mc, slot_ids, ctr, recs, depths);
        return;
    }
    const uint32_t grid = persistent_grid(n_hint, PROJ_THREADS, PROJ_MIN_CTAS, sm_count);
    const uint32_t g = group & ~ENTITY_MODES;
    with_layout_degree(g & 1u ? CloudLayout::F16 : CloudLayout::F32, g >> 1, [&](auto L, auto Dt) {
        constexpr CloudLayout Lv = decltype(L)::value;
        constexpr uint32_t D = decltype(Dt)::value;
        if constexpr (!is_4d(Lv)) {
            auto* kernel = (group & ENTITY_MODES) ? project_many_kernel<is_f16(Lv), D, true>
                                                  : project_many_kernel<is_f16(Lv), D, false>;
            kernel<<<grid, PROJ_THREADS, 0, stream>>>(tab, group, need_sh ? 1u : 0u, mc, slot_ids, ctr, recs, extra, cutoff_tab);
        }
    });
}

void launch_depth_range_views(const SceneTable& tab, uint32_t v, uint32_t n_view, const uint32_t* sorted_payload,
                              const uint32_t* slot_ids, const FrameCounters* ctr, ViewRanges* view_ranges, uint32_t n_hint,
                              int sm_count, cudaStream_t stream) {
    const uint32_t grid = persistent_grid(n_hint, DRV_THREADS, DRV_CTAS_PER_SM, sm_count);
    depth_range_views_kernel<<<grid, DRV_THREADS, 0, stream>>>(tab, v, n_view, sorted_payload, slot_ids, ctr, view_ranges);
}

void launch_project_4d_scene(const SceneTable& tab, const SceneTimes& times, const SceneClasses& classes,
                             const ModeConsts& mc, const uint32_t* slot_ids, const FrameCounters* ctr, SplatRec* recs,
                             float* depths, uint32_t n_hint, int sm_count, cudaStream_t stream) {
    const uint32_t grid = persistent_grid(n_hint, PROJ_THREADS, PROJ_MIN_CTAS, sm_count);
    project_4d_scene_kernel<<<grid, PROJ_THREADS, 0, stream>>>(tab, times, classes, mc, slot_ids, ctr, recs, depths);
}

void launch_depth_range(const float4* pos, uint32_t n, const uint32_t* sorted_payload, const uint32_t* slot_ids,
                        FrameCounters* ctr, const FrameConsts& fc, cudaStream_t stream) {
    depth_range_kernel<<<1, 32, 0, stream>>>(pos, n, sorted_payload, slot_ids, ctr, fc);
}

void launch_project(CloudLayout layout, uint32_t sh_degree, const void* blocks, const uint32_t* index_list, int by_slot, const FrameCounters* ctr,
                    const FrameConsts& fc, SplatRec* recs, float4* extra, uint32_t n_hint, int sm_count,
                    const float* cutoff_tab, float4* aux, const ModeConsts* modes, cudaStream_t stream) {
    // a persistent grid: as many CTAs as the launch bound lets the SMs hold, fewer when the hint (last frame's visible
    // count + head-room) has less than one group of 32 entries for each warp; the loop strides, so any n_vis is correct
    const uint32_t grid = persistent_grid(n_hint, PROJ_THREADS, PROJ_MIN_CTAS, sm_count);
    // (both f16 layouts run the F16 kernels: the covariance record differs only in fc.cov_pre)
    with_layout_degree(layout, sh_degree, [&](auto L, auto Dt) {
        constexpr CloudLayout Lv = decltype(L)::value;
        constexpr uint32_t D = decltype(Dt)::value;
        if constexpr (!is_4d(Lv)) {
            if (modes)   // Classification / OpticalFlow (no aux outputs)
                project_modes_kernel<is_f16(Lv), D><<<grid, PROJ_THREADS, 0, stream>>>(blocks, index_list, by_slot, ctr, fc, *modes,
                                                                                      recs, extra, cutoff_tab);
            else
                project_kernel<is_f16(Lv), D><<<grid, PROJ_THREADS, 0, stream>>>(blocks, index_list, by_slot, ctr, fc, recs, extra,
                                                                                cutoff_tab, aux);
        }
    });
}

}  // namespace bgs
