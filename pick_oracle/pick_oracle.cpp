// CPU oracle of bgs_render_entities_pick's pick frame (include/bgs.h).  TEST INFRASTRUCTURE ONLY.
//
// Input: a frame as entity_oracle computes it -- records by front-to-back rank (12 floats: cx, cy, ux, uy, vx, vy, bbox x,
// bbox y, r, g, b, opacity), each rank's blend kind (0 quad-uv, 1 conic, 2 surfel; | 4 when its entity draws its bounding
// box), the surfel extras of each rank (16 floats, eo_frame_ex's surfel_extra; needed when some rank is a surfel), the tile
// ranges and slices (ranks), each rank's splat depth d, and the scene's depth buffer (or none).  For every pixel the
// oracle walks its tile's slice in blend order and lists every pair that blends: the pair's rank, its weight w = a T
// evaluated in f64 (T from 1 by T *= 1 - a; an overlay edge pair: w = T, then T = 0), and a bound on |w_f32 - w| of
// the kernel, from the per-alpha relative error (c0 + c1 |power|) U the caller passes (tests/blend_cases.py) and the
// f32 roundings of the T updates (a pair whose exponential is below FLT_MIN: w itself, the kernel may flush it to 0).
// The walk stops once T < 1e-4.  near_stop[pixel] marks pixels where some T the walk compared lay within its own bound
// of 1e-4 (the kernel may blend one pair more or less there).
//
// Coverage: the kernels' f32 decisions, bit for bit (raster.cu: quad_uv with the fma on the dy term; the conic's |m| <= R
// and power <= 0; the surfel's |m| <= e0.x, then the homography hu x hv, us, vs and power = -0.5 min(s3, s2) <= 0, its
// overlay on m / e0.x), after the record's bbox (lo | hi << 16) test against the pixel's 8x4 warp rectangle, and d >=
// the pixel's scene depth when a buffer is given.  A frame with a surfel rank and no surfel extras is refused (-1).
#include <cmath>
#include <cstdint>
#include <cstring>

namespace {
constexpr double U = 1.0 / 16777216.0;
constexpr float T_STOP = 1.0e-4f;
constexpr double FLT_MIN_NORMAL = 1.1754943508222875e-38;   // 2^-126

bool box_edge(float u, float v) {
    const float sx = u * 0.5f + 0.5f, sy = v * 0.5f + 0.5f;
    return sx < 0.08f || sx > 1.0f - 0.08f || sy < 0.08f || sy > 1.0f - 0.08f;
}

// raster.cu's surfel branch (raster_body, kind 2) at pixel centre (fx, fy) for record q and extras e (e0..e3): the
// coverage |m| <= e0.x (the depth test, which the caller makes, comes next), then the power; false where not covered or
// power > 0.  mx, my: the quad-space offset; R = e0.x.
bool surfel_decide(const float* q, const float* e, float fx, float fy, float& mx, float& my, float& R, float& power) {
    const float dx = fx - q[0], dy = fy - q[1];
    mx = dx + dx; my = -(dy + dy); R = e[0];
    if (!(std::fabs(mx) <= R && std::fabs(my) <= R)) return false;
    const float pcx = mx + e[1], pcy = my * e[3] + e[2];
    const float* T0 = e + 4; const float* T1 = e + 8; const float* T2 = e + 12;
    const float hux = pcx * T2[0] - T0[0], huy = pcx * T2[1] - T0[1], huz = pcx * T2[2] - T0[2];
    const float hvx = pcy * T2[0] - T1[0], hvy = pcy * T2[1] - T1[1], hvz = pcy * T2[2] - T1[2];
    const float cpx = huy * hvz - huz * hvy, cpy = huz * hvx - hux * hvz, cpz = hux * hvy - huy * hvx;
    const float us = cpx / cpz, vs = cpy / cpz;
    const float s3 = us * us + vs * vs;
    const float ex = e[1] - pcx, ey = e[2] - pcy;
    const float s2 = 2.0f * (ex * ex + ey * ey);
    power = -(0.5f * std::fmin(s3, s2));
    return !(power > 0.0f);
}
}  // namespace

extern "C" {

// Pass 1 (pairs == NULL): counts[pixel] = pairs listed at the pixel.  Pass 2: offsets (H*W + 1, from pass 1's counts)
// and the outputs, pair-major: rank, w, bound.
int po_pick(uint32_t W, uint32_t H, uint32_t n_vis, const float* recs, const uint8_t* kinds, const float* surfel_extra,
            const uint32_t* tile_ranges, const uint32_t* tile_entries, const float* splat_d,
            const float* scene /* H x W or NULL */, double c0, double c1, uint32_t* counts, const uint64_t* offsets,
            uint32_t* pair_rank, double* pair_w, double* pair_bound, uint8_t* near_stop) {
    for (uint32_t r = 0; r < n_vis; ++r)
        if ((kinds[r] & 3) > 2 || ((kinds[r] & 3) == 2 && !surfel_extra)) return -1;
    const uint32_t tiles_x = (W + 15) / 16;
    for (uint32_t py = 0; py < H; ++py)
        for (uint32_t px = 0; px < W; ++px) {
            const size_t pix = (size_t)py * W + px;
            const uint32_t tile = (py / 16) * tiles_x + px / 16;
            const float fx = (float)px + 0.5f, fy = (float)py + 0.5f;
            const float zs = scene ? scene[pix] : 0.0f;
            const int wx0 = (int)(px & ~7u), wy0 = (int)(py & ~3u);   // the pixel's warp rectangle (raster_body)
            double T = 1.0, sens = 0.0;   // sens: sum over earlier pairs of a / (1 - a) x their alpha's relative error
            uint32_t cnt = 0;
            bool near = false;
            for (uint32_t e = tile_ranges[2 * tile]; e < tile_ranges[2 * tile + 1]; ++e) {
                const uint32_t r = tile_entries[e];
                const float* q = recs + (size_t)r * 12;
                uint32_t bx, by;
                memcpy(&bx, q + 6, 4); memcpy(&by, q + 7, 4);
                if ((int)(bx >> 16) < wx0 || (int)(bx & 0xFFFFu) > wx0 + 7 || (int)(by >> 16) < wy0 ||
                    (int)(by & 0xFFFFu) > wy0 + 3)
                    continue;   // (the warp's candidate test: the bbox misses its 8x4 pixels)
                const int kind = kinds[r] & 3;
                const bool box = (kinds[r] & 4) != 0;
                double power;
                bool edge = false;
                if (kind == 0) {
                    const float dx = fx - q[0], dy = fy - q[1];
                    const float u = std::fmaf(q[3], dy, q[2] * dx), v = std::fmaf(q[5], dy, q[4] * dx);
                    if (!(std::fabs(u) <= 1.0f && std::fabs(v) <= 1.0f)) continue;
                    if (scene && !(splat_d[r] >= zs)) continue;
                    edge = box && box_edge(u, v);
                    power = -4.5 * (double)std::fmaf(v, v, u * u);
                } else if (kind == 2) {
                    float mx, my, R, pf;
                    if (!surfel_decide(q, surfel_extra + (size_t)r * 16, fx, fy, mx, my, R, pf)) {
                        // (coverage failed, or power > 0: either way the pair does not blend; the depth test sits
                        // between the two in the kernel, which changes nothing here)
                        continue;
                    }
                    if (scene && !(splat_d[r] >= zs)) continue;
                    edge = box && box_edge(mx / R, my / R);
                    power = (double)pf;
                } else {
                    const float dx = fx - q[0], dy = fy - q[1];
                    const float mx = dx + dx, my = -(dy + dy), R = q[5];
                    if (!(std::fabs(mx) <= R && std::fabs(my) <= R)) continue;
                    if (scene && !(splat_d[r] >= zs)) continue;
                    const float ddx = -mx, ddy = -my;
                    const float t1 = (q[2] * ddx) * ddx, t2 = (q[4] * ddy) * ddy;
                    const float pf = (-0.5f * (t1 + t2)) + ((q[3] * ddx) * ddy);
                    if (pf > 0.0f) continue;
                    edge = box && box_edge(mx / R, my / R);
                    power = (double)pf;
                }
                double w, bound;
                if (edge) {
                    w = T;
                    bound = T * (sens + (cnt + 2) * U);   // the kernel's T against this one
                } else {
                    const double a = std::fmin(std::exp(power) * (double)q[11], 0.999);
                    const double da = (c0 + c1 * std::fabs(power)) * U;
                    w = a * T;
                    bound = w * (da + sens + (cnt + 3) * U);
                    // the kernels' exponentials (ex2.approx.ftz, __expf) flush results below FLT_MIN to 0: such a pair
                    // may blend with w = 0 (surfel powers reach far below ln FLT_MIN at their quad's corners)
                    if (std::exp(power) < FLT_MIN_NORMAL) bound = std::fmax(bound, w);
                    if (a < 0.999) sens += a / (1.0 - a) * da;
                }
                if (pair_rank) {
                    const uint64_t o = offsets[pix] + cnt;
                    pair_rank[o] = r; pair_w[o] = w; pair_bound[o] = bound;
                }
                ++cnt;
                T = edge ? 0.0 : T - w;
                const double tb2 = T * (sens + (cnt + 2) * U);
                if (std::fabs(T - (double)T_STOP) <= tb2 + 1e-12) near = true;
                if (T < (double)T_STOP) break;
            }
            if (!pair_rank) counts[pix] = cnt;
            else near_stop[pix] = near ? 1 : 0;
        }
    return 0;
}

// The surfel decisions of pick frames per pair, for comparing with entity_oracle's: record recs[j] (12 floats) and its
// extras extra[j] (16 floats) at the pixel centre (pixel_xy[2j], pixel_xy[2j+1]): covered[j] (coverage and power <= 0,
// no depth test) and edge[j] (covered and on the overlay's edge band).
int po_surfel_probe(uint32_t count, const float* recs, const float* extra, const float* pixel_xy, uint8_t* covered,
                    uint8_t* edge) {
    for (uint32_t j = 0; j < count; ++j) {
        float mx, my, R, pf;
        const bool c = surfel_decide(recs + (size_t)j * 12, extra + (size_t)j * 16, pixel_xy[2 * j], pixel_xy[2 * j + 1], mx,
                                     my, R, pf);
        covered[j] = c ? 1u : 0u;
        edge[j] = c && box_edge(mx / R, my / R) ? 1u : 0u;
    }
    return 0;
}

}  // extern "C"
