// depth_oracle.cpp -- see depth_oracle.h.  The oracle's translation unit is compiled into this one, so the walks below
// reuse its projection, sort, binning and coverage decision (decide / alpha_of) unchanged; only the depth test is new.
#include "../oracle/bgs_oracle.cpp"

#include "depth_oracle.h"

namespace {

// include/bgs.h: d = pz / pw with (pz, pw) the z and w lanes of world_to_clip(model * pos), each divided by w + 1e-9
float splat_depth_of(const float* p, const orc_view& v, const orc_uniform& u) {
    float pw[4], c[4];
    mat4_point(u.transform, p[0], p[1], p[2], pw);
    mat4_point(v.clip_from_world, pw[0], pw[1], pw[2], c);
    const float den = c[3] + 0.000000001f;
    const float pz = c[2] / den, pwl = c[3] / den;
    return pz / pwl;
}

// the test at pixel (x, y): d >= scene (IEEE: a NaN on either side fails); no buffer passes everything
struct Scene {
    const float* z;
    uint64_t pitch;
    bool pass(float d, int x, int y) const {
        if (!z) return true;
        const float s = *reinterpret_cast<const float*>(reinterpret_cast<const char*>(z) + (uint64_t)y * pitch + 4u * (uint64_t)x);
        return d >= s;
    }
};

// rank -> d of the frame's visible splats
std::vector<float> rank_depths(const Ctx& C, const Frame& F, const float* pos) {
    std::vector<float> d(F.n_vis);
    for (uint32_t r = 0; r < F.n_vis; ++r) d[r] = splat_depth_of(pos + 4 * (size_t)F.rank_to_id[r], *C.v, *C.u);
    return d;
}

}  // namespace

extern "C" {

int dor_splat_depth(uint32_t n, const float* pos_vis, const orc_view* view, const orc_uniform* u, uint32_t count,
                    const uint32_t* ids, float* out) {
    if (!view || !u) return 2;
    for (uint32_t j = 0; j < count; ++j) {
        if (ids[j] >= n) return 3;
        out[j] = splat_depth_of(pos_vis + 4 * (size_t)ids[j], *view, *u);
    }
    return 0;
}

// orc_render_ref_over's back-to-front pass, literally as the reference's pipeline runs it: each fragment is depth-tested
// against the (never written) scene depth before it is blended
int dor_render_ref_over(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                        const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* dst_init,
                        const float* scene, uint64_t pitch_bytes, float* out, int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_frame(C, n, pos_vis, sh, rot, so, F);
    const std::vector<float> dz = rank_depths(C, F, pos_vis);
    const Scene Z{scene, pitch_bytes};
    const int W = C.Wi, H = C.Hi;
    const int band = 8;
    const int nb = (H + band - 1) / band;
#pragma omp parallel for schedule(dynamic, 1)
    for (int b = 0; b < nb; ++b) {
        const int y0 = b * band, y1 = std::min(H, y0 + band) - 1;
        for (int y = y0; y <= y1; ++y) for (int x = 0; x < W; ++x) {
            float* px = out + 4 * ((size_t)y * W + x);
            if (dst_init) {
                const float* d = dst_init + 4 * ((size_t)y * W + x);
                px[0] = d[0]; px[1] = d[1]; px[2] = d[2]; px[3] = d[3];
            } else {
                px[0] = 0.0f; px[1] = 0.0f; px[2] = 0.0f; px[3] = 1.0f;
            }
        }
        for (int64_t r = (int64_t)F.n_vis - 1; r >= 0; --r) {   // far -> near
            const orc_splat& sp = F.splats[r];
            if (sp.xlo > sp.xhi || sp.yhi < y0 || sp.ylo > y1) continue;
            const int ya = std::max(sp.ylo, y0), yb = std::min(sp.yhi, y1);
            for (int y = ya; y <= yb; ++y) for (int x = sp.xlo; x <= sp.xhi; ++x) {
                float a;
                if (!eval_alpha(sp, *s, (float)x + 0.5f, (float)y + 0.5f, &a)) continue;
                if (!Z.pass(dz[r], x, y)) continue;
                float* px = out + 4 * ((size_t)y * W + x);
                const float ia = 1.0f - a;
                px[0] = sp.r * a + ia * px[0];
                px[1] = sp.g * a + ia * px[1];
                px[2] = sp.b * a + ia * px[2];
                px[3] = a + ia * px[3];
            }
        }
    }
    return 0;
}

int dor_render_tiles(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                     const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* scene,
                     uint64_t pitch_bytes, float* out, int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_frame(C, n, pos_vis, sh, rot, so, F);
    const std::vector<float> dz = rank_depths(C, F, pos_vis);
    const Scene Z{scene, pitch_bytes};
    const int W = C.Wi, H = C.Hi;
    const int TX = (W + TILE - 1) / TILE, TY = (H + TILE - 1) / TILE;
    std::vector<uint64_t> count;
    std::vector<uint32_t> entries;
    bin_tiles(F, TX, TY, count, entries);
#pragma omp parallel for schedule(dynamic, 4)
    for (int t = 0; t < TX * TY; ++t) {
        const int tx = t % TX, ty = t / TX;
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
            for (uint64_t e = count[t]; e < count[t + 1]; ++e) {
                const orc_splat& sp = F.splats[entries[e]];
                float a;
                if (!eval_alpha(sp, *s, (float)x + 0.5f, (float)y + 0.5f, &a)) continue;
                if (!Z.pass(dz[entries[e]], x, y)) continue;
                const float w = a * T;
                cr += w * sp.r; cg += w * sp.g; cb += w * sp.b;
                T = T * (1.0f - a);
                if (T < T_STOP) break;
            }
            float* px = out + 4 * ((size_t)y * W + x);
            px[0] = cr; px[1] = cg; px[2] = cb; px[3] = 1.0f;
        }
    }
    return 0;
}

int dor_blend_trace(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                    const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* scene,
                    uint64_t pitch_bytes, orc_trace* out, int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_frame(C, n, pos_vis, sh, rot, so, F);
    const std::vector<float> dz = rank_depths(C, F, pos_vis);
    const Scene Z{scene, pitch_bytes};
    const int W = C.Wi, H = C.Hi;
    const int TX = (W + TILE - 1) / TILE, TY = (H + TILE - 1) / TILE;
    std::vector<uint64_t> count;
    std::vector<uint32_t> entries;
    bin_tiles(F, TX, TY, count, entries);
#pragma omp parallel for schedule(dynamic, 4)
    for (int t = 0; t < TX * TY; ++t) {
        const int tx = t % TX, ty = t / TX;
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            orc_trace o;
            std::memset(&o, 0, sizeof(o));
            o.rank0 = o.rank1 = -1;
            o.stop_margin = std::numeric_limits<double>::infinity();
            float T = 1.0f;
            double T64 = 1.0, c64[3] = {0.0, 0.0, 0.0};
            for (uint64_t e = count[t]; e < count[t + 1]; ++e) {
                const orc_splat& sp = F.splats[entries[e]];
                const Decision d = decide(sp, *s, (float)x + 0.5f, (float)y + 0.5f);
                if (!d.covered || !Z.pass(dz[entries[e]], x, y)) continue;
                // from here on: orc_blend_trace's step
                const float x32 = std::exp(d.power) * sp.op, a = std::fmin(x32, 0.999f);
                const double a64 = std::fmin(std::exp((double)d.power) * (double)sp.op, 0.999);
                const double w64 = a64 * T64;
                o.w_power += w64 * std::fabs((double)d.power);
                c64[0] += w64 * sp.r; c64[1] += w64 * sp.g; c64[2] += w64 * sp.b;
                T64 *= 1.0 - a64;
                if (o.n_blended == 0) o.rank0 = (int32_t)entries[e];
                else if (o.n_blended == 1) o.rank1 = (int32_t)entries[e];
                ++o.n_blended;
                o.max_c = std::fmax(o.max_c, std::fmax(std::fabs(sp.r), std::fmax(std::fabs(sp.g), std::fabs(sp.b))));
                o.max_power = std::fmax(o.max_power, std::fabs(d.power));
                if (std::fabs(x32 - 0.999f) <= 1.0e-5f * 0.999f) o.flags |= ORC_TRACE_NEAR_CLAMP;
                if (x32 < 0.999f) {
                    o.flags |= ORC_TRACE_UNCLAMPED;
                    o.t_sens += (double)a / (1.0 - (double)a);
                    o.t_sens_power += (double)a / (1.0 - (double)a) * std::fabs((double)d.power);
                }
                T = T * (1.0f - a);
                const double margin = std::fabs((double)T / (double)T_STOP - 1.0);
                o.stop_margin = std::fmin(o.stop_margin, margin);
                if (margin <= 1.0e-5) o.flags |= ORC_TRACE_NEAR_STOP;
                if (T < T_STOP) break;
            }
            o.c64[0] = c64[0]; o.c64[1] = c64[1]; o.c64[2] = c64[2];
            o.T64 = T64;
            o.T = T;
            out[(size_t)y * W + x] = o;
        }
    }
    return 0;
}

int dor_coverage_probe(uint32_t count, const orc_splat* splats, const orc_settings* s, const float* pixel_xy,
                       const float* splat_d, const float* scene_d, orc_probe* out) {
    const int rc = orc_coverage_probe(count, splats, s, pixel_xy, out);
    if (rc != 0 || !splat_d) return rc;
    for (uint32_t j = 0; j < count; ++j) {
        if (splat_d[j] >= scene_d[j]) continue;
        out[j].covered = 0u;
        out[j].covered_if_unfused = 0u;
        out[j].alpha = 0.0f;
    }
    return 0;
}

}  // extern "C"
