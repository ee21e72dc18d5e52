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
