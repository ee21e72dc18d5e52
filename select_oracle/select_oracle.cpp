// select_oracle.cpp -- CPU oracle of SparseSelect; see select_oracle.h.  Built with -ffp-contract=off (FP policy).
#include "select_oracle.h"

#include <cmath>
#include <cstring>
#include <vector>

#include <omp.h>

namespace {

// ---- restated from bevy_gaussian_splatting_b200/csrc/select.cu (cell and bucket functions) ----
constexpr double SEL_CLAMP = 1099511627776.0;   // 2^40
long long cell_coord(float p, double cell) {
    double q = (double)p / cell;
    q = q < -SEL_CLAMP ? -SEL_CLAMP : (q > SEL_CLAMP ? SEL_CLAMP : q);
    return (long long)std::floor(q);
}
double cell_size(float radius) { return (double)radius * (1.0 + 1.0 / 1024.0); }
constexpr unsigned long long HX = 0x9E3779B97F4A7C15ull, HY = 0xC2B2AE3D27D4EB4Full, HZ = 0x165667B19E3779F9ull;
unsigned long long cell_lin(long long cx, long long cy, long long cz) {
    return (unsigned long long)cx * HX + (unsigned long long)cy * HY + (unsigned long long)cz * HZ;
}
uint32_t bucket_of(unsigned long long h, uint32_t mask) {
    h ^= h >> 29;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 32;
    return (uint32_t)h & mask;
}
uint32_t num_buckets(uint32_t n) {
    uint32_t b = 1u << 10;
    while (b < n && b < (1u << 24)) b <<= 1;
    return b;
}
bool finite3(const float* p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// the definition's test: d2 = ((dx*dx + dy*dy) + dz*dz) < r2, f32, no contraction
inline bool within(const float* a, const float* b, float r2) {
    const float dx = b[0] - a[0], dy = b[1] - a[1], dz = b[2] - a[2];
    const float d2 = (dx * dx + dy * dy) + dz * dz;
    return d2 < r2;
}

bool bad_radius(float radius) { return !(radius >= 0.0f) || std::isinf(radius); }

void finish(uint32_t n, const std::vector<uint32_t>& cnt, uint32_t threshold, uint8_t* mask, uint32_t* out_selected) {
    uint32_t sel = 0;
    for (uint32_t i = 0; i < n; ++i) {
        mask[i] = cnt[i] < threshold ? 1 : 0;
        sel += mask[i];
    }
    if (out_selected) *out_selected = sel;
}

}  // namespace

extern "C" {

int orc_select_sparse(uint32_t n, const float* pos, float radius, uint32_t threshold, uint8_t* mask, uint32_t* out_selected,
                      int threads) {
    if (bad_radius(radius)) return -1;
    const float r2 = radius * radius;
    std::vector<uint32_t> cnt(n, 0u);
    if (threads > 0) omp_set_num_threads(threads);
#pragma omp parallel for schedule(dynamic, 64)
    for (long long i = 0; i < (long long)n; ++i) {
        uint32_t c = 0;
        for (uint32_t j = 0; j < n; ++j) c += within(pos + 4 * i, pos + 4 * (size_t)j, r2) ? 1u : 0u;
        cnt[i] = c;
    }
    finish(n, cnt, threshold, mask, out_selected);
    return 0;
}

uint32_t orc_select_buckets(uint32_t n, const float* pos, float radius, uint32_t* out_bucket, int64_t* out_cell3) {
    const uint32_t nb = num_buckets(n);
    const double cell = cell_size(radius);
    for (uint32_t i = 0; i < n; ++i) {
        const float* p = pos + 4 * (size_t)i;
        long long c[3] = {0, 0, 0};
        uint32_t b = nb;
        if (finite3(p)) {
            for (int k = 0; k < 3; ++k) c[k] = cell_coord(p[k], cell);
            b = bucket_of(cell_lin(c[0], c[1], c[2]), nb - 1u);
        }
        if (out_bucket) out_bucket[i] = b;
        if (out_cell3)
            for (int k = 0; k < 3; ++k) out_cell3[3 * (size_t)i + k] = c[k];
    }
    return nb;
}

int orc_select_sparse_grid(uint32_t n, const float* pos, float radius, uint32_t threshold, uint8_t* mask, uint32_t* out_selected,
                           int threads) {
    if (bad_radius(radius)) return -1;
    const float r2 = radius * radius;
    std::vector<uint32_t> cnt(n, 0u);
    if (threshold == 0u || r2 == 0.0f) {   // nothing can reach a threshold of 0; nothing is below a zero r2
        finish(n, cnt, threshold, mask, out_selected);
        return 0;
    }
    std::vector<uint32_t> bucket(n);
    const uint32_t nb = orc_select_buckets(n, pos, radius, bucket.data(), nullptr);
    // counting sort by bucket (stable): start[b] .. start[b + 1]
    std::vector<uint32_t> start((size_t)nb + 2, 0u), order(n);
    for (uint32_t i = 0; i < n; ++i) ++start[(size_t)bucket[i] + 1];
    for (size_t b = 0; b <= nb; ++b) start[b + 1] += start[b];
    {
        std::vector<uint32_t> at(start.begin(), start.end() - 1);
        for (uint32_t i = 0; i < n; ++i) order[at[bucket[i]]++] = i;
    }
    const double cell = cell_size(radius);
    if (threads > 0) omp_set_num_threads(threads);
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i) {
        const float* p = pos + 4 * (size_t)i;
        if (!finite3(p)) continue;   // count 0
        const long long cx = cell_coord(p[0], cell), cy = cell_coord(p[1], cell), cz = cell_coord(p[2], cell);
        uint32_t b[27];
        uint32_t c = 0;
        for (int k = 0; k < 27; ++k) {
            b[k] = bucket_of(cell_lin(cx - 1 + k % 3, cy - 1 + k / 3 % 3, cz - 1 + k / 9), nb - 1u);
            bool dup = false;
            for (int m = 0; m < k; ++m) dup |= b[m] == b[k];
            if (dup) continue;
            for (uint32_t s = start[b[k]]; s < start[(size_t)b[k] + 1] && c < threshold; ++s)
                c += within(p, pos + 4 * (size_t)order[s], r2) ? 1u : 0u;
        }
        cnt[i] = c;
    }
    finish(n, cnt, threshold, mask, out_selected);
    return 0;
}

}  // extern "C"

// ---- point in mesh (src/query/raycast.rs:54-124) ----------------------------------------------------------------
namespace {

struct V3 {
    float x, y, z;
};
V3 sub(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
// glam's scalar Vec3 order: dot = (x x' + y y') + z z', cross = (y z' - y' z, z x' - z' x, x y' - x' y)
float dot(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
V3 cross(V3 a, V3 b) { return {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; }
constexpr float MS_EPS = 0.000001f;

// raycast.rs:92-124, the definition
bool ray_hits(V3 o, V3 v0, V3 v1, V3 v2) {
    const V3 dir = {1.0f, 0.0f, 0.0f};
    const V3 e1 = sub(v1, v0), e2 = sub(v2, v0);
    const V3 h = cross(dir, e2);
    const float a = dot(e1, h);
    if (a > -MS_EPS && a < MS_EPS) return false;
    const float f = 1.0f / a;
    const V3 s = sub(o, v0);
    const float u = f * dot(s, h);
    if (!(u >= 0.0f && u <= 1.0f)) return false;
    const V3 q = cross(s, e1);
    const float v = f * dot(dir, q);
    if (v < 0.0f || u + v > 1.0f) return false;
    const float t = f * dot(e2, q);
    return t > MS_EPS;
}

V3 xform(const float* m, const float* p) {   // column-major m, ((m_r0 x + m_r1 y) + m_r2 z) + m_r3
    return {((m[0] * p[0] + m[4] * p[1]) + m[8] * p[2]) + m[12], ((m[1] * p[0] + m[5] * p[1]) + m[9] * p[2]) + m[13],
            ((m[2] * p[0] + m[6] * p[1]) + m[10] * p[2]) + m[14]};
}
const float kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
V3 vert(const float* v, uint32_t i) { return {v[3 * (size_t)i], v[3 * (size_t)i + 1], v[3 * (size_t)i + 2]}; }
bool bad_mesh(uint32_t nv, const float* verts, uint32_t nt, const uint32_t* idx) {
    if (nt > 0 && (!verts || !idx)) return true;
    for (size_t k = 0; k < (size_t)nt * 3; ++k)
        if (idx[k] >= nv) return true;
    return false;
}
uint32_t finish_mask(uint32_t n, const std::vector<uint32_t>& hits, uint8_t* mask) {
    uint32_t in = 0;
    for (uint32_t i = 0; i < n; ++i) {
        mask[i] = hits[i] & 1u;
        in += mask[i];
    }
    return in;
}

// ---- restated from bevy_gaussian_splatting_b200/csrc/mesh_select.cu (setup, classes, slack, grid ladder, cells) ----
constexpr float MS_FAR = 4611686018427387904.0f;
constexpr double MS_KAPPA_MAX = 65536.0;
constexpr int MS_LEVELS = 13;
constexpr uint32_t MS_MAX_DIM = 4096;
bool ms_near(float x) { return std::fabs(x) < MS_FAR; }

struct Rec {
    V3 v0, e1, e2, h;
    float f;
};
bool rec_hit(V3 o, const Rec& r) {
    const V3 dir = {1.0f, 0.0f, 0.0f};
    const V3 s = sub(o, r.v0);
    const float u = r.f * dot(s, r.h);
    if (!(u >= 0.0f && u <= 1.0f)) return false;
    const V3 q = cross(s, r.e1);
    const float v = r.f * dot(dir, q);
    if (v < 0.0f || u + v > 1.0f) return false;
    return r.f * dot(r.e2, q) > MS_EPS;
}
bool mesh_box(V3 v0, V3 v1, V3 v2, V3 e1, V3 e2, float a, double* box) {
    if (!(ms_near(v0.x) && ms_near(v0.y) && ms_near(v0.z) && ms_near(v1.x) && ms_near(v1.y) && ms_near(v1.z) && ms_near(v2.x) &&
          ms_near(v2.y) && ms_near(v2.z)))
        return false;
    const double E = std::fmax(std::fmax(std::fabs((double)e1.y), std::fabs((double)e1.z)),
                               std::fmax(std::fabs((double)e2.y), std::fabs((double)e2.z)));
    const double kappa = E * E / std::fabs((double)a);
    if (!(kappa <= MS_KAPPA_MAX)) return false;
    const double ylo = std::fmin(std::fmin((double)v0.y, (double)v1.y), (double)v2.y);
    const double yhi = std::fmax(std::fmax((double)v0.y, (double)v1.y), (double)v2.y);
    const double zlo = std::fmin(std::fmin((double)v0.z, (double)v1.z), (double)v2.z);
    const double zhi = std::fmax(std::fmax((double)v0.z, (double)v1.z), (double)v2.z);
    const double m = std::fmax(std::fmax(std::fabs(ylo), std::fabs(yhi)), std::fmax(std::fabs(zlo), std::fabs(zhi)));
    const double slack = (kappa + 1.0) * E * (1.0 / 131072.0) + m * (1.0 / 1073741824.0) + 1e-30;
    box[0] = ylo - slack;
    box[1] = yhi + slack;
    box[2] = zlo - slack;
    box[3] = zhi + slack;
    return true;
}
uint32_t mesh_cell(double p, double p0, double inv, uint32_t n) {
    const double c = std::floor((p - p0) * inv);
    return c < 0.0 ? 0u : (c >= (double)n ? n - 1u : (uint32_t)c);
}
struct Grid {
    double y0, z0, inv_y, inv_z;
    uint32_t ny, nz;
};

struct MeshPlan {
    std::vector<Rec> bin, glob;
    std::vector<double> box;   // 4 per binned record
    double y0 = 0, y1 = 0, z0 = 0, z1 = 0;
    std::vector<Grid> levels;
    std::vector<uint64_t> level_pairs;
    int level = -1;
};

MeshPlan plan_mesh(const float* verts, uint32_t nt, const uint32_t* idx) {
    MeshPlan P;
    for (uint32_t t = 0; t < nt; ++t) {
        const V3 v0 = vert(verts, idx[3 * (size_t)t]), v1 = vert(verts, idx[3 * (size_t)t + 1]), v2 = vert(verts, idx[3 * (size_t)t + 2]);
        const V3 e1 = sub(v1, v0), e2 = sub(v2, v0);
        const V3 h = cross({1.0f, 0.0f, 0.0f}, e2);
        const float a = dot(e1, h);
        if ((a > -MS_EPS && a < MS_EPS) || !std::isfinite(a)) continue;
        const Rec r = {v0, e1, e2, h, 1.0f / a};
        double b[4];
        if (mesh_box(v0, v1, v2, e1, e2, a, b)) {
            P.bin.push_back(r);
            P.box.insert(P.box.end(), b, b + 4);
        } else {
            P.glob.push_back(r);
        }
    }
    const uint32_t nb = (uint32_t)P.bin.size();
    if (nb == 0) return P;
    P.y0 = P.z0 = INFINITY;
    P.y1 = P.z1 = -INFINITY;
    for (uint32_t b = 0; b < nb; ++b) {
        P.y0 = std::fmin(P.y0, P.box[4 * b]);
        P.y1 = std::fmax(P.y1, P.box[4 * b + 1]);
        P.z0 = std::fmin(P.z0, P.box[4 * b + 2]);
        P.z1 = std::fmax(P.z1, P.box[4 * b + 3]);
    }
    const double W = P.y1 - P.y0, H = P.z1 - P.z0;
    const double side = std::sqrt(W * H / (2.0 * (double)nb));
    auto dim = [&](double ext) {
        const double d = std::ceil(ext / side);
        return d >= (double)MS_MAX_DIM ? MS_MAX_DIM : (d >= 1.0 ? (uint32_t)d : 1u);
    };
    const uint32_t ny0 = side > 0.0 ? dim(W) : 1u, nz0 = side > 0.0 ? dim(H) : 1u;
    for (int l = 0; l < MS_LEVELS; ++l) {
        Grid g;
        g.ny = ny0 >> l ? ny0 >> l : 1u;
        g.nz = nz0 >> l ? nz0 >> l : 1u;
        g.y0 = P.y0;
        g.z0 = P.z0;
        g.inv_y = (double)g.ny / W;
        g.inv_z = (double)g.nz / H;
        uint64_t pairs = 0;
        for (uint32_t b = 0; b < nb; ++b) {
            const double* x = &P.box[4 * (size_t)b];
            pairs += (uint64_t)(mesh_cell(x[1], g.y0, g.inv_y, g.ny) - mesh_cell(x[0], g.y0, g.inv_y, g.ny) + 1u) *
                     (mesh_cell(x[3], g.z0, g.inv_z, g.nz) - mesh_cell(x[2], g.z0, g.inv_z, g.nz) + 1u);
        }
        P.levels.push_back(g);
        P.level_pairs.push_back(pairs);
        if (g.ny == 1u && g.nz == 1u) break;
    }
    const uint64_t budget = (1ull << 24) + 4ull * nb;
    int l = 0;
    while (l + 1 < (int)P.levels.size() && P.level_pairs[l] > budget) ++l;
    P.level = l;
    return P;
}

}  // namespace

extern "C" {

int orc_select_in_mesh(uint32_t n, const float* pos_vis, uint32_t nv, const float* verts, uint32_t nt, const uint32_t* idx,
                       const float* mesh_from_cloud, uint8_t* mask, uint32_t* out_inside, int threads) {
    if (bad_mesh(nv, verts, nt, idx)) return -1;
    const float* M = mesh_from_cloud ? mesh_from_cloud : kIdentity;
    std::vector<uint32_t> hits(n, 0u);
    if (threads > 0) omp_set_num_threads(threads);
#pragma omp parallel for schedule(dynamic, 64)
    for (long long i = 0; i < (long long)n; ++i) {
        const V3 o = xform(M, pos_vis + 4 * i);
        uint32_t c = 0;
        for (uint32_t t = 0; t < nt; ++t)
            c += ray_hits(o, vert(verts, idx[3 * (size_t)t]), vert(verts, idx[3 * (size_t)t + 1]), vert(verts, idx[3 * (size_t)t + 2]))
                     ? 1u : 0u;
        hits[i] = c;
    }
    const uint32_t in = finish_mask(n, hits, mask);
    if (out_inside) *out_inside = in;
    return 0;
}

int orc_select_in_mesh_grid(uint32_t n, const float* pos_vis, uint32_t nv, const float* verts, uint32_t nt, const uint32_t* idx,
                            const float* mesh_from_cloud, uint8_t* mask, uint32_t* out_inside, int threads) {
    if (bad_mesh(nv, verts, nt, idx)) return -1;
    const float* M = mesh_from_cloud ? mesh_from_cloud : kIdentity;
    const MeshPlan P = plan_mesh(verts, nt, idx);
    const uint32_t nb = (uint32_t)P.bin.size();
    // counting sort of the (cell, triangle) pairs by cell
    Grid g{};
    std::vector<uint32_t> start(1, 0u), tri;
    if (P.level >= 0) {
        g = P.levels[P.level];
        const size_t cells = (size_t)g.ny * g.nz;
        start.assign(cells + 1, 0u);
        std::vector<uint32_t> keys, vals;
        for (uint32_t b = 0; b < nb; ++b) {
            const double* x = &P.box[4 * (size_t)b];
            for (uint32_t z = mesh_cell(x[2], g.z0, g.inv_z, g.nz); z <= mesh_cell(x[3], g.z0, g.inv_z, g.nz); ++z)
                for (uint32_t y = mesh_cell(x[0], g.y0, g.inv_y, g.ny); y <= mesh_cell(x[1], g.y0, g.inv_y, g.ny); ++y) {
                    keys.push_back(z * g.ny + y);
                    vals.push_back(b);
                }
        }
        for (uint32_t k : keys) ++start[(size_t)k + 1];
        for (size_t c = 0; c < cells; ++c) start[c + 1] += start[c];
        tri.resize(keys.size());
        std::vector<uint32_t> at(start.begin(), start.end() - 1);
        for (size_t k = 0; k < keys.size(); ++k) tri[at[keys[k]]++] = vals[k];
    }
    std::vector<uint32_t> hits(n, 0u);
    if (threads > 0) omp_set_num_threads(threads);
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i) {
        const V3 q = xform(M, pos_vis + 4 * i);
        uint32_t c = 0;
        if (std::isfinite(q.x) && std::isfinite(q.y) && std::isfinite(q.z)) {
            if (!(ms_near(q.x) && ms_near(q.y) && ms_near(q.z))) {
                for (uint32_t b = 0; b < nb; ++b) c += rec_hit(q, P.bin[b]) ? 1u : 0u;
            } else if (nb && (double)q.y >= P.y0 && (double)q.y <= P.y1 && (double)q.z >= P.z0 && (double)q.z <= P.z1) {
                const size_t cell = (size_t)mesh_cell(q.z, g.z0, g.inv_z, g.nz) * g.ny + mesh_cell(q.y, g.y0, g.inv_y, g.ny);
                for (uint32_t s = start[cell]; s < start[cell + 1]; ++s) c += rec_hit(q, P.bin[tri[s]]) ? 1u : 0u;
            }
            for (const Rec& r : P.glob) c += rec_hit(q, r) ? 1u : 0u;
        }
        hits[i] = c;
    }
    const uint32_t in = finish_mask(n, hits, mask);
    if (out_inside) *out_inside = in;
    return 0;
}

int orc_mesh_plan(uint32_t nv, const float* verts, uint32_t nt, const uint32_t* idx, uint32_t* out_counts, int32_t* out_level,
                  uint64_t* out_pairs) {
    if (bad_mesh(nv, verts, nt, idx)) return -1;
    const MeshPlan P = plan_mesh(verts, nt, idx);
    out_counts[0] = (uint32_t)P.bin.size();
    out_counts[1] = (uint32_t)P.glob.size();
    out_counts[2] = P.level >= 0 ? P.levels[P.level].ny : 0u;
    out_counts[3] = P.level >= 0 ? P.levels[P.level].nz : 0u;
    *out_level = P.level;
    *out_pairs = P.level >= 0 ? P.level_pairs[P.level] : 0u;
    return 0;
}

// The binned boxes (4 doubles each, ylo yhi zlo zhi) in triangle order, NaN rows for the dropped and global ones.
int orc_mesh_boxes(uint32_t nv, const float* verts, uint32_t nt, const uint32_t* idx, double* out_box, int32_t* out_class) {
    if (bad_mesh(nv, verts, nt, idx)) return -1;
    for (uint32_t t = 0; t < nt; ++t) {
        const V3 v0 = vert(verts, idx[3 * (size_t)t]), v1 = vert(verts, idx[3 * (size_t)t + 1]), v2 = vert(verts, idx[3 * (size_t)t + 2]);
        const V3 e1 = sub(v1, v0), e2 = sub(v2, v0);
        const float a = dot(e1, cross({1.0f, 0.0f, 0.0f}, e2));
        double* b = out_box + 4 * (size_t)t;
        b[0] = b[1] = b[2] = b[3] = NAN;
        if ((a > -MS_EPS && a < MS_EPS) || !std::isfinite(a)) out_class[t] = 0;
        else out_class[t] = mesh_box(v0, v1, v2, e1, e2, a, b) ? 1 : 2;
    }
    return 0;
}

}  // extern "C"
