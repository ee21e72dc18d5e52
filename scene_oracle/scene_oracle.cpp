// scene_oracle.cpp -- see scene_oracle.h.  The oracle's translation unit is compiled into this one, so the joint frame
// below keys, projects, bins and blends with its functions unchanged; only the joint index space is new.
#include "../oracle/bgs_oracle.cpp"

#include "scene_oracle.h"

namespace {

struct Scene {
    std::vector<uint32_t> offset;        // o_j, and N at [k]
    std::vector<orc_settings> settings;  // the frame's settings with cloud j's cov_pre bit
    std::vector<Ctx> ctx;                // the oracle's context of cloud j (its uniform)
    uint32_t seg(uint32_t g) const {
        return (uint32_t)(std::upper_bound(offset.begin(), offset.end() - 1, g) - offset.begin()) - 1u;
    }
};

bool make_scene(Scene& S, uint32_t k, const sor_cloud* cl, const orc_view* v, const orc_settings* s) {
    if (k == 0 || !cl || !v || !s) return false;
    S.offset.assign(k + 1, 0u);
    S.settings.assign(k, *s);
    S.ctx.resize(k);
    for (uint32_t j = 0; j < k; ++j) {
        S.offset[j + 1] = S.offset[j] + cl[j].n;
        S.settings[j].reserved = (s->reserved & ~1u) | (cl[j].cov_pre ? 1u : 0u);
        if (!make_ctx(S.ctx[j], v, &cl[j].u, &S.settings[j])) return false;
    }
    return true;
}

// build_frame over the joint index space
void build_scene_frame(const Scene& S, const sor_cloud* cl, const orc_view& v, const orc_settings& s, Frame& F) {
    const uint32_t n = S.offset.back();
    const uint32_t shift = S.ctx[0].plan.shift;
    F.keys.resize(n); F.order.resize(n);
#pragma omp parallel for schedule(static)
    for (int64_t g = 0; g < (int64_t)n; ++g) {
        const uint32_t j = S.seg((uint32_t)g), i = (uint32_t)g - S.offset[j];
        F.keys[g] = key_of(cl[j].pos_vis + 4 * (size_t)i, v, cl[j].u, shift).key;
    }
    std::iota(F.order.begin(), F.order.end(), 0u);
    const uint32_t* kp = F.keys.data();
    std::stable_sort(F.order.begin(), F.order.end(), [kp](uint32_t a, uint32_t b) { return kp[a] < kp[b]; });
    uint32_t nv = 0;
    const uint32_t culled = 0xFFFFFFFFu >> shift;
    while (nv < n && F.keys[F.order[nv]] != culled) ++nv;
    F.n_vis = nv;
    F.splats.resize(nv); F.rank_to_id.resize(nv);
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)nv; ++r) {
        const uint32_t g = F.order[nv - 1 - r], j = S.seg(g);
        const size_t i = g - S.offset[j];
        F.rank_to_id[r] = g;
        project_one(S.ctx[j], cl[j].pos_vis + 4 * i, cl[j].sh + 48 * i, cl[j].rot + 4 * i, cl[j].scale_opacity + 4 * i, F.splats[r]);
    }
    if (s.rasterize_mode == 1u && n >= 2) {   // build_frame's Depth rule over the joint list, each from its own cloud
        auto dist = [&](uint32_t g) {
            const uint32_t j = S.seg(g);
            float pw[4];
            const float* p = cl[j].pos_vis + 4 * (size_t)(g - S.offset[j]);
            mat4_point(cl[j].u.transform, p[0], p[1], p[2], pw);
            const float d[3] = {pw[0] - v.world_position[0], pw[1] - v.world_position[1], pw[2] - v.world_position[2]};
            return std::sqrt(dot3(d, d));
        };
        const float dmin = dist(F.order[n - 1]), dmax = dist(F.order[1]);
        for (uint32_t r = 0; r < nv; ++r) {
            if (F.splats[r].xlo > F.splats[r].xhi) continue;
            const uint32_t g = F.rank_to_id[r], j = S.seg(g);
            float rgb[3];
            depth_to_rgb(dist(g), dmin, dmax, rgb);
            if (!(s.draw_mode == 2u && cl[j].pos_vis[4 * (size_t)(g - S.offset[j]) + 3] > 0.5f)) {
                F.splats[r].r = rgb[0]; F.splats[r].g = rgb[1]; F.splats[r].b = rgb[2];
            }
        }
    }
}

}  // namespace

extern "C" {

int sor_sorted_entries(uint32_t k, const sor_cloud* clouds, const orc_view* view, uint32_t depth_bits, uint32_t* out) {
    orc_settings s{};
    s.gaussian_mode = 1u;
    s.radix_sort_depth_bits = depth_bits;
    Scene S;
    if (!make_scene(S, k, clouds, view, &s)) return 2;
    const uint32_t n = S.offset.back(), shift = S.ctx[0].plan.shift;
    std::vector<uint32_t> keys(n), order(n);
    for (uint32_t g = 0; g < n; ++g) {
        const uint32_t j = S.seg(g);
        keys[g] = key_of(clouds[j].pos_vis + 4 * (size_t)(g - S.offset[j]), *view, clouds[j].u, shift).key;
    }
    orc_stable_sort(n, keys.data(), order.data());
    for (uint32_t e = 0; e < n; ++e) { out[2 * e] = keys[order[e]]; out[2 * e + 1] = order[e]; }
    return 0;
}

int sor_render_tiles(uint32_t k, const sor_cloud* clouds, const orc_view* view, const orc_settings* s, float* out,
                     uint32_t* tile_ranges, uint32_t* tile_entries, uint64_t cap, uint64_t* n_pairs, uint32_t* n_vis,
                     uint32_t* rank_to_id, orc_splat* records, int threads) {
    Scene S;
    if (!make_scene(S, k, clouds, view, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_scene_frame(S, clouds, *view, *s, F);
    const int W = S.ctx[0].Wi, H = S.ctx[0].Hi;
    const int TX = (W + TILE - 1) / TILE, TY = (H + TILE - 1) / TILE, NT = TX * TY;
    std::vector<uint64_t> count;
    std::vector<uint32_t> entries;
    bin_tiles(F, TX, TY, count, entries);
    const uint64_t total = count[NT];
    if (n_pairs) *n_pairs = total;
    if (n_vis) *n_vis = F.n_vis;
    if (rank_to_id) std::memcpy(rank_to_id, F.rank_to_id.data(), (size_t)F.n_vis * 4);
    if (records) std::memcpy(records, F.splats.data(), (size_t)F.n_vis * sizeof(orc_splat));
    if (tile_ranges) for (int t = 0; t < NT; ++t) {
        const bool empty = count[t] == count[t + 1];
        tile_ranges[2 * t] = empty ? 0u : (uint32_t)count[t];
        tile_ranges[2 * t + 1] = empty ? 0u : (uint32_t)count[t + 1];
    }
    if (tile_entries) std::memcpy(tile_entries, entries.data(), (size_t)std::min<uint64_t>(total, cap) * 4);
    if (!out) return 0;
#pragma omp parallel for schedule(dynamic, 4)
    for (int t = 0; t < NT; ++t) {   // orc_render_tiles' walk
        const int tx = t % TX, ty = t / TX;
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
            for (uint64_t e = count[t]; e < count[t + 1]; ++e) {
                const orc_splat& sp = F.splats[entries[e]];
                float a;
                if (!eval_alpha(sp, *s, (float)x + 0.5f, (float)y + 0.5f, &a)) continue;
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

int sor_render_ref_over(uint32_t k, const sor_cloud* clouds, const orc_view* view, const orc_settings* s, const float* dst_init,
                        float* out, int threads) {
    Scene S;
    if (!make_scene(S, k, clouds, view, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_scene_frame(S, clouds, *view, *s, F);
    const int W = S.ctx[0].Wi, H = S.ctx[0].Hi;
    const int band = 8, nb = (H + band - 1) / band;
#pragma omp parallel for schedule(dynamic, 1)
    for (int b = 0; b < nb; ++b) {   // orc_render_ref_over's pass
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
        for (int64_t r = (int64_t)F.n_vis - 1; r >= 0; --r) {
            const orc_splat& sp = F.splats[r];
            if (sp.xlo > sp.xhi || sp.yhi < y0 || sp.ylo > y1) continue;
            const int ya = std::max(sp.ylo, y0), yb = std::min(sp.yhi, y1);
            for (int y = ya; y <= yb; ++y) for (int x = sp.xlo; x <= sp.xhi; ++x) {
                float a;
                if (!eval_alpha(sp, *s, (float)x + 0.5f, (float)y + 0.5f, &a)) continue;
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

}  // extern "C"
