// mesh_select.cu -- point-in-mesh selection (src/query/raycast.rs:54-124) on the device-resident cloud: a gaussian is
// inside a triangle mesh iff the ray from its position along +x hits an odd number of triangles, each hit decided by
// the reference's literal f32 Moller-Trumbore test (ray_intersects_triangle).
//
// The ray runs along +x, so whether a triangle can be hit depends on the point only through (y, z): the candidates
// of a point are found on a uniform 2D grid over (y, z), and every candidate is decided by the literal test:
//   1. mesh_setup_kernel, one thread per triangle: v0, edge1, edge2, h, a and f exactly as the test computes them
//      (they do not depend on the point, so precomputing them is bit-identical).  Triangles the `a` test rejects, or
//      whose `a` is not finite, can never be hit and are dropped.  A survivor gets a 64 B record and a class:
//        binned -- a yz box that contains every point the f32 test can accept (the slack, see mesh_box);
//        global -- no such box is derived (a sliver, a vertex at or beyond 2^62, a non-finite vertex): the triangle
//                  is tested against every point;
//   2. mesh_levels_kernel: the (cell, triangle) pair count of each grid resolution of a ladder (the host picks the
//      finest one whose pairs fit the budget, see mesh_plan_levels);
//   3. mesh_emit_kernel: one (cell, triangle) pair per cell each binned box overlaps; the stable radix sort of
//      radix.cu orders them by cell and its `ranges` epilogue yields each cell's slice (the parity count does not
//      depend on the order within a cell);
//   4. mesh_count_kernel, one thread per gaussian: q = mesh_from_cloud * (x, y, z, 1), its one cell, the literal test
//      over that cell's triangles and over the global ones, and the visibility lane per mode in both device copies.
//      A point whose q is not finite is never hit; a point with a coordinate at or beyond 2^62 is tested against
//      every survivor (no box bounds its rounding, see mesh_box).
//
// Cost: O(T) setup and pair emission, one radix sort of the pairs, and a count of O(N x (triangles per cell +
// global triangles)).  A closed mesh covers its yz silhouette about twice, so a cell holds a few triangles.
#include "common.cuh"
#include "launch.cuh"

namespace bgs {

constexpr int MS_THREADS = 256;
constexpr float MS_EPS = 0.000001f;              // raycast.rs:93
constexpr float MS_FAR = 4611686018427387904.0f;   // 2^62: |coordinates| below it cannot overflow the test's f32 products
constexpr double MS_KAPPA_MAX = 65536.0;           // binned triangles: E^2 / |a| <= 2^16 (mesh_box)
constexpr int MS_LEVELS = 13;                      // grid resolutions 4096 >> L per axis, L = 0..12
constexpr uint32_t MS_MAX_DIM = 4096;

struct MeshRec {
    float4 v0f;   // v0, f = 1 / a
    float4 e1;    // edge1
    float4 e2;    // edge2
    float4 h;     // h = dir x edge2 (general expression)
};

// The per-call device words (zeroed per call).  The grid bounds are f64 kept as order-preserving u64 keys under
// atomicMax: [0] -ylo, [1] yhi, [2] -zlo, [3] zhi of the union of the binned boxes.
struct MeshWords {
    uint32_t n_bin, n_glob, n_pairs, inside;
    uint32_t barrier, pad[3];
    unsigned long long bound[4];
    unsigned long long level_pairs[MS_LEVELS];
};

struct MeshGrid {
    double y0, z0, inv_y, inv_z;   // cell(p) = floor((p - p0) * inv), clamped to [0, n - 1]
    uint32_t ny, nz;
};
struct MeshLevels {
    MeshGrid g[MS_LEVELS];
    int n;
};

// ---- the box and cell functions.  select_oracle/select_oracle.cpp restates them (test infrastructure) ----------
//
// The slack.  For a triangle with finite vertices below 2^62 and a point q below 2^62, nothing in the test overflows,
// h = (+-0, -e2z, e2y) exactly, s.x * h.x = +-0, and 0 * q'.y, 0 * q'.z are +-0: u and v depend on (q.y, q.z) only,
//   u = fl(f * fl(fl(s.y * -e2z) + fl(s.z * e2y))),   v = fl(f * fl(fl(s.y * e1z) - fl(e1y * s.z))),   s = fl(q - v0).
// Let uu = 2^-24, E = max(|e1y|, |e1z|, |e2y|, |e2z|), A the exact e1z e2y - e1y e2z and kappa = E^2 / |A|.  Each of
// a, s.h and q'.x carries at most two roundings of terms bounded by E^2 (a) or 2 |s| E (the others), so
// |a - A| <= 4 uu E^2 = 4 uu kappa |A|, and with U, V the exact barycentrics of s (s = U e1 + V e2 in yz, |s| <=
// (|U| + |V|) E), an accepted u, v in [0, 1] gives |U - u|, |V - v| <= delta with
//   delta <= (12 uu kappa + 3 uu) / (1 - 8 uu kappa) <= 1.04 (12 uu kappa + 3 uu)   for kappa <= 1.02 * 2^16.
// So (U, V) lies within l1 distance 5 delta of the exact triangle, s within 5 delta E of its box (each component),
// and q = v0 + s up to the roundings of s and of e1, e2 (3 uu E).  With kappa computed from the f32 a
// (kappa_hat <= 2^16 gives kappa <= 1.02 kappa_hat), every accepted point lies within
//   (64 kappa_hat + 19) uu E  <=  2^-17 (kappa_hat + 1) E
// of the vertices' yz box: that is the slack, a factor 2 over the bound.  2^-30 max|y, z| covers the f64 rounding of
// the box (an f32 triangle with a nonzero yz area has E >= 2^-24 max|y, z|), and 1e-30 the subnormal products.
// A triangle with kappa_hat > 2^16 (a sliver: u and v are dominated by rounding, and an accepted point may lie far
// along its edges) is global.  An exact bound is the contract here, the numbers measured by random probing (a few
// tens of uu E) sit well inside it.
__host__ __device__ __forceinline__ bool ms_near(float x) { return fabsf(x) < MS_FAR; }   // false for NaN

__host__ __device__ __forceinline__ bool mesh_box(float3 v0, float3 v1, float3 v2, float3 e1, float3 e2, float a, double* box) {
    if (!(ms_near(v0.x) && ms_near(v0.y) && ms_near(v0.z) && ms_near(v1.x) && ms_near(v1.y) && ms_near(v1.z) &&
          ms_near(v2.x) && ms_near(v2.y) && ms_near(v2.z)))
        return false;
    const double E = fmax(fmax(fabs((double)e1.y), fabs((double)e1.z)), fmax(fabs((double)e2.y), fabs((double)e2.z)));
    const double kappa = E * E / fabs((double)a);
    if (!(kappa <= MS_KAPPA_MAX)) return false;
    const double ylo = fmin(fmin((double)v0.y, (double)v1.y), (double)v2.y), yhi = fmax(fmax((double)v0.y, (double)v1.y), (double)v2.y);
    const double zlo = fmin(fmin((double)v0.z, (double)v1.z), (double)v2.z), zhi = fmax(fmax((double)v0.z, (double)v1.z), (double)v2.z);
    const double m = fmax(fmax(fabs(ylo), fabs(yhi)), fmax(fabs(zlo), fabs(zhi)));
    const double slack = (kappa + 1.0) * E * (1.0 / 131072.0) + m * (1.0 / 1073741824.0) + 1e-30;
    box[0] = ylo - slack;
    box[1] = yhi + slack;
    box[2] = zlo - slack;
    box[3] = zhi + slack;
    return true;
}

// One monotone f64 function of the coordinate, for boxes and points alike: a point inside a box lands in one of
// the box's cells.
__host__ __device__ __forceinline__ uint32_t mesh_cell(double p, double p0, double inv, uint32_t n) {
    const double c = floor((p - p0) * inv);
    return c < 0.0 ? 0u : (c >= (double)n ? n - 1u : (uint32_t)c);
}

__device__ __forceinline__ unsigned long long ms_key(double d) {   // order-preserving u64 of a (non-NaN) double
    const unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// ---- the literal test (raycast.rs:92-124) over a precomputed record, glam's scalar Vec3 order, f32 RNE, no FMA ----
__device__ __forceinline__ float ms_dot(float ax, float ay, float az, float bx, float by, float bz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
}
__device__ __forceinline__ bool ms_hit(float3 q, const MeshRec& r) {
    const float f = r.v0f.w;
    const float sx = __fsub_rn(q.x, r.v0f.x), sy = __fsub_rn(q.y, r.v0f.y), sz = __fsub_rn(q.z, r.v0f.z);
    const float u = __fmul_rn(f, ms_dot(sx, sy, sz, r.h.x, r.h.y, r.h.z));
    if (!(u >= 0.0f && u <= 1.0f)) return false;
    // q' = s x edge1
    const float qx = __fsub_rn(__fmul_rn(sy, r.e1.z), __fmul_rn(r.e1.y, sz));
    const float qy = __fsub_rn(__fmul_rn(sz, r.e1.x), __fmul_rn(r.e1.z, sx));
    const float qz = __fsub_rn(__fmul_rn(sx, r.e1.y), __fmul_rn(r.e1.x, sy));
    const float v = __fmul_rn(f, ms_dot(1.0f, 0.0f, 0.0f, qx, qy, qz));
    if (v < 0.0f || __fadd_rn(u, v) > 1.0f) return false;
    const float t = __fmul_rn(f, ms_dot(r.e2.x, r.e2.y, r.e2.z, qx, qy, qz));
    return t > MS_EPS;
}

__device__ __forceinline__ float3 ms_vertex(const float* __restrict__ v, uint32_t i) {
    return make_float3(__ldg(v + 3 * (size_t)i), __ldg(v + 3 * (size_t)i + 1), __ldg(v + 3 * (size_t)i + 2));
}
__device__ __forceinline__ float3 ms_sub(float3 a, float3 b) {
    return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}

__global__ void __launch_bounds__(MS_THREADS) mesh_setup_kernel(const float* __restrict__ verts, const uint32_t* __restrict__ idx,
                                                                uint32_t nt, MeshRec* __restrict__ bin_rec, double4* __restrict__ bin_box,
                                                                MeshRec* __restrict__ glob_rec, MeshWords* __restrict__ w) {
    const uint32_t t = blockIdx.x * MS_THREADS + threadIdx.x;
    bool binned = false;
    double box[4] = {0.0, 0.0, 0.0, 0.0};
    if (t < nt) {
        const float3 v0 = ms_vertex(verts, __ldg(idx + 3 * (size_t)t)), v1 = ms_vertex(verts, __ldg(idx + 3 * (size_t)t + 1)),
                     v2 = ms_vertex(verts, __ldg(idx + 3 * (size_t)t + 2));
        const float3 e1 = ms_sub(v1, v0), e2 = ms_sub(v2, v0);
        // h = dir x edge2 with dir = (1, 0, 0), the general expression (0 * inf = NaN must stay NaN)
        const float hx = __fsub_rn(__fmul_rn(0.0f, e2.z), __fmul_rn(e2.y, 0.0f));
        const float hy = __fsub_rn(__fmul_rn(0.0f, e2.x), __fmul_rn(e2.z, 1.0f));
        const float hz = __fsub_rn(__fmul_rn(1.0f, e2.y), __fmul_rn(e2.x, 0.0f));
        const float a = ms_dot(e1.x, e1.y, e1.z, hx, hy, hz);
        // a NaN never passes the u test (f, u NaN); a = +-inf gives f = +-0 and t = +-0 or NaN, never > eps
        if (!(a > -MS_EPS && a < MS_EPS) && isfinite(a)) {
            MeshRec r;
            r.v0f = make_float4(v0.x, v0.y, v0.z, __fdiv_rn(1.0f, a));
            r.e1 = make_float4(e1.x, e1.y, e1.z, 0.0f);
            r.e2 = make_float4(e2.x, e2.y, e2.z, 0.0f);
            r.h = make_float4(hx, hy, hz, 0.0f);
            if (mesh_box(v0, v1, v2, e1, e2, a, box)) {
                const uint32_t slot = atomicAdd(&w->n_bin, 1u);
                bin_rec[slot] = r;
                bin_box[slot] = make_double4(box[0], box[1], box[2], box[3]);
                binned = true;
            } else {
                glob_rec[atomicAdd(&w->n_glob, 1u)] = r;
            }
        }
    }
    // the grid bounds: per-warp maxima of the four keys, one atomic per warp
    unsigned long long k[4] = {0ull, 0ull, 0ull, 0ull};
    if (binned) {
        k[0] = ms_key(-box[0]);
        k[1] = ms_key(box[1]);
        k[2] = ms_key(-box[2]);
        k[3] = ms_key(box[3]);
    }
    const bool any = __any_sync(0xffffffffu, binned);
    if (!any) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, k[j], o);
            k[j] = other > k[j] ? other : k[j];
        }
    }
    if ((threadIdx.x & 31) == 0)
        for (int j = 0; j < 4; ++j) atomicMax(&w->bound[j], k[j]);
}

__device__ __forceinline__ unsigned long long ms_box_cells(const double4& b, const MeshGrid& g, uint32_t& y0, uint32_t& y1,
                                                           uint32_t& z0, uint32_t& z1) {
    y0 = mesh_cell(b.x, g.y0, g.inv_y, g.ny);
    y1 = mesh_cell(b.y, g.y0, g.inv_y, g.ny);
    z0 = mesh_cell(b.z, g.z0, g.inv_z, g.nz);
    z1 = mesh_cell(b.w, g.z0, g.inv_z, g.nz);
    return (unsigned long long)(y1 - y0 + 1u) * (z1 - z0 + 1u);
}

__global__ void __launch_bounds__(MS_THREADS) mesh_levels_kernel(const double4* __restrict__ bin_box, uint32_t n_bin, MeshLevels L,
                                                                 MeshWords* __restrict__ w) {
    const uint32_t t = blockIdx.x * MS_THREADS + threadIdx.x;
    double4 b = make_double4(0.0, 0.0, 0.0, 0.0);
    if (t < n_bin) b = bin_box[t];
    for (int l = 0; l < L.n; ++l) {
        uint32_t y0, y1, z0, z1;
        unsigned long long c = t < n_bin ? ms_box_cells(b, L.g[l], y0, y1, z0, z1) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(&w->level_pairs[l], c);
    }
}

__global__ void __launch_bounds__(MS_THREADS) mesh_emit_kernel(const double4* __restrict__ bin_box, uint32_t n_bin, MeshGrid g,
                                                               uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                               MeshWords* __restrict__ w) {
    const uint32_t t = blockIdx.x * MS_THREADS + threadIdx.x;
    if (t >= n_bin) return;
    uint32_t y0, y1, z0, z1;
    const uint32_t cnt = (uint32_t)ms_box_cells(bin_box[t], g, y0, y1, z0, z1);
    uint32_t k = atomicAdd(&w->n_pairs, cnt);
    for (uint32_t z = z0; z <= z1; ++z)
        for (uint32_t y = y0; y <= y1; ++y, ++k) {
            keys[k] = z * g.ny + y;
            vals[k] = t;
        }
}

struct MeshXform {
    float m[16];   // mesh_from_cloud, column-major
};

// One thread per gaussian.  mode 0 (replace): lane = inside ? 1 : 0; mode 1 (add): lane = 1 where inside, else untouched.
__global__ void __launch_bounds__(MS_THREADS) mesh_count_kernel(CloudView cloud, uint32_t n, MeshXform M,
                                                                const MeshRec* __restrict__ bin_rec, uint32_t n_bin,
                                                                const MeshRec* __restrict__ glob_rec, uint32_t n_glob,
                                                                const uint32_t* __restrict__ cell_tri, const uint2* __restrict__ ranges,
                                                                MeshGrid g, double y1, double z1, uint32_t mode,
                                                                uint32_t* __restrict__ inside_count) {
    const uint32_t i = blockIdx.x * MS_THREADS + threadIdx.x;
    bool inside = false;
    if (i < n) {
        const float4 p = __ldg(cloud.pos + i);
        const float* m = M.m;
        // q = M (x, y, z, 1): ((m_r0 x + m_r1 y) + m_r2 z) + m_r3 per row r
        float3 q;
        q.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], p.x), __fmul_rn(m[4], p.y)), __fmul_rn(m[8], p.z)), m[12]);
        q.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[1], p.x), __fmul_rn(m[5], p.y)), __fmul_rn(m[9], p.z)), m[13]);
        q.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[2], p.x), __fmul_rn(m[6], p.y)), __fmul_rn(m[10], p.z)), m[14]);
        uint32_t hits = 0;
        // a non-finite q is never hit: inf * 0 or inf - inf makes u NaN, or inf * h makes it infinite
        if (isfinite(q.x) && isfinite(q.y) && isfinite(q.z)) {
            if (!(ms_near(q.x) && ms_near(q.y) && ms_near(q.z))) {
                for (uint32_t b = 0; b < n_bin; ++b) hits += ms_hit(q, bin_rec[b]) ? 1u : 0u;
            } else if (n_bin && (double)q.y >= g.y0 && (double)q.y <= y1 && (double)q.z >= g.z0 && (double)q.z <= z1) {
                const uint32_t c = mesh_cell((double)q.z, g.z0, g.inv_z, g.nz) * g.ny + mesh_cell((double)q.y, g.y0, g.inv_y, g.ny);
                const uint2 r = __ldg(ranges + c);   // (~start, end); (0, 0) = empty
                for (uint32_t s = ~r.x; s < r.y; ++s) hits += ms_hit(q, bin_rec[__ldg(cell_tri + s)]) ? 1u : 0u;
            }
            for (uint32_t b = 0; b < n_glob; ++b) hits += ms_hit(q, glob_rec[b]) ? 1u : 0u;
        }
        inside = (hits & 1u) != 0u;
        if (mode == 0u || inside) cloud.store_visibility(i, inside ? 1.0f : 0.0f);
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, inside);
    if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(inside_count, (uint32_t)__popc(ballot));
}

// ---- host side -----------------------------------------------------------------------------------------------------
static uint32_t ms_grid(uint32_t n) { return (n + MS_THREADS - 1) / MS_THREADS; }
static double ms_unkey(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
    double d;
    memcpy(&d, &b, 8);
    return d;
}

size_t mesh_words_bytes() { return sizeof(MeshWords); }
size_t mesh_rec_bytes() { return sizeof(MeshRec); }

void launch_mesh_setup(const float* verts, const uint32_t* idx, uint32_t nt, void* bin_rec, void* bin_box, void* glob_rec, void* words,
                       cudaStream_t stream) {
    if (nt == 0) return;
    mesh_setup_kernel<<<ms_grid(nt), MS_THREADS, 0, stream>>>(verts, idx, nt, static_cast<MeshRec*>(bin_rec),
                                                              static_cast<double4*>(bin_box), static_cast<MeshRec*>(glob_rec),
                                                              static_cast<MeshWords*>(words));
}

// The grid ladder over the union of the binned boxes (bounds from the setup's words): level 0 aims at 2 cells per
// binned triangle in square cells, at most 4096 per axis; level l halves each axis l times (down to 1 x 1).  Depends
// on the triangles only.  select_oracle/select_oracle.cpp restates it.
static MeshLevels mesh_plan_levels(const unsigned long long bound[4], uint32_t n_bin) {
    MeshLevels L{};
    const double y0 = -ms_unkey(bound[0]), y1 = ms_unkey(bound[1]), z0 = -ms_unkey(bound[2]), z1 = ms_unkey(bound[3]);
    const double W = y1 - y0, H = z1 - z0;
    const double side = sqrt(W * H / (2.0 * (double)n_bin));
    auto dim = [&](double ext) {
        const double d = ceil(ext / side);
        return d >= (double)MS_MAX_DIM ? MS_MAX_DIM : (d >= 1.0 ? (uint32_t)d : 1u);
    };
    const uint32_t ny0 = side > 0.0 ? dim(W) : 1u, nz0 = side > 0.0 ? dim(H) : 1u;
    for (int l = 0; l < MS_LEVELS; ++l) {
        MeshGrid& g = L.g[l];
        g.ny = ny0 >> l ? ny0 >> l : 1u;
        g.nz = nz0 >> l ? nz0 >> l : 1u;
        g.y0 = y0;
        g.z0 = z0;
        g.inv_y = (double)g.ny / W;
        g.inv_z = (double)g.nz / H;
        L.n = l + 1;
        if (g.ny == 1u && g.nz == 1u) break;
    }
    return L;
}

// The pair budget: 2^24 + 4 per binned triangle (the 1 x 1 level, n_bin pairs, always fits).
static uint64_t mesh_pair_budget(uint32_t n_bin) { return (1ull << 24) + 4ull * n_bin; }

// Level counts for the ladder of a setup whose words are back on the host (`words_host`).
void launch_mesh_levels(const void* bin_box, const void* words_host, void* words, cudaStream_t stream) {
    const MeshWords* wh = static_cast<const MeshWords*>(words_host);
    const MeshLevels L = mesh_plan_levels(wh->bound, wh->n_bin);
    mesh_levels_kernel<<<ms_grid(wh->n_bin), MS_THREADS, 0, stream>>>(static_cast<const double4*>(bin_box), wh->n_bin, L,
                                                                      static_cast<MeshWords*>(words));
}

// After the level counts are back: the finest level within the budget -> its pairs and cells.
void mesh_pick_level(const void* words_host, int* level, uint64_t* pairs, uint32_t* cells) {
    const MeshWords* wh = static_cast<const MeshWords*>(words_host);
    const MeshLevels L = mesh_plan_levels(wh->bound, wh->n_bin);
    int l = 0;
    while (l + 1 < L.n && wh->level_pairs[l] > mesh_pair_budget(wh->n_bin)) ++l;
    *level = l;
    *pairs = wh->level_pairs[l];
    *cells = L.g[l].ny * L.g[l].nz;
}

void launch_mesh_emit(const void* bin_box, const void* words_host, int level, uint32_t* keys, uint32_t* vals, void* words,
                      cudaStream_t stream) {
    const MeshWords* wh = static_cast<const MeshWords*>(words_host);
    const MeshLevels L = mesh_plan_levels(wh->bound, wh->n_bin);
    mesh_emit_kernel<<<ms_grid(wh->n_bin), MS_THREADS, 0, stream>>>(static_cast<const double4*>(bin_box), wh->n_bin, L.g[level], keys,
                                                                    vals, static_cast<MeshWords*>(words));
}

uint32_t* mesh_words_pairs(void* words) { return &static_cast<MeshWords*>(words)->n_pairs; }
uint32_t* mesh_words_barrier(void* words) { return &static_cast<MeshWords*>(words)->barrier; }
uint32_t* mesh_words_inside(void* words) { return &static_cast<MeshWords*>(words)->inside; }
uint32_t mesh_words_n_bin(const void* words_host) { return static_cast<const MeshWords*>(words_host)->n_bin; }

// level < 0: no binned triangle (no grid)
void launch_mesh_count(CloudView cloud, uint32_t n, const float* mesh_from_cloud, const void* bin_rec, const void* glob_rec,
                       const uint32_t* cell_tri, const uint2* ranges, const void* words_host, int level, uint32_t mode, void* words,
                       cudaStream_t stream) {
    if (n == 0) return;
    const MeshWords* wh = static_cast<const MeshWords*>(words_host);
    MeshXform M;
    memcpy(M.m, mesh_from_cloud, sizeof(M.m));
    MeshGrid g{};
    double y1 = 0.0, z1 = 0.0;
    if (level >= 0) {
        g = mesh_plan_levels(wh->bound, wh->n_bin).g[level];
        y1 = ms_unkey(wh->bound[1]);
        z1 = ms_unkey(wh->bound[3]);
    }
    mesh_count_kernel<<<ms_grid(n), MS_THREADS, 0, stream>>>(cloud, n, M, static_cast<const MeshRec*>(bin_rec), level >= 0 ? wh->n_bin : 0u,
                                                             static_cast<const MeshRec*>(glob_rec), wh->n_glob, cell_tri, ranges, g, y1,
                                                             z1, mode, &static_cast<MeshWords*>(words)->inside);
}

}  // namespace bgs
