// entity_oracle.cpp -- see entity_oracle.h.  scene4d_oracle.cpp (the temporal and 3D oracles with it) is compiled into
// this translation unit, so every per-gaussian rule, binning and coverage decision below is theirs unchanged; only the
// per-cloud settings are new.
#include "../scene4d_oracle/scene4d_oracle.cpp"

#include "entity_oracle.h"

extern "C" {

int eo_frame(uint32_t k, const s4o_cloud* cl, const orc_view* view, const orc_settings* es, const uint32_t* nc,
             const tor_temporal* ex, const float* scene, uint64_t pitch_bytes, uint32_t* n_vis, uint64_t* n_pairs, uint32_t* sorted,
             float* records, uint32_t* rank_to_id, float* depths, uint32_t* tile_ranges, uint32_t* tile_entries, uint64_t cap,
             float* image, int threads) {
    if (k == 0 || !cl || !view || !es || !nc || !ex) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    // per cloud: its own settings (4D: Gaussian4d; 3D: its cov_pre bit), context, times and num_classes
    std::vector<orc_settings> st(es, es + k);
    std::vector<Ctx> ctx(k);
    std::vector<tor_temporal> tp(k, *ex);
    std::vector<uint32_t> offset(k + 1, 0u);
    for (uint32_t j = 0; j < k; ++j) {
        offset[j + 1] = offset[j] + cl[j].n;
        st[j].radix_sort_depth_bits = es[0].radix_sort_depth_bits;
        tp[j].num_classes = nc[j];
        if (cl[j].kind == 1u) {
            st[j].gaussian_mode = 2u;
            tp[j].time_start = cl[j].time_start;
            tp[j].time_stop = cl[j].time_stop;
        } else {
            if (st[j].rasterize_mode == 4u || st[j].rasterize_mode == 5u) return 3;
            st[j].reserved = (es[j].reserved & ~1u) | (cl[j].cov_pre ? 1u : 0u);
        }
        if (!make_ctx(ctx[j], view, &cl[j].u, &st[j])) return 2;
    }
    auto seg = [&](uint32_t g) { return (uint32_t)(std::upper_bound(offset.begin(), offset.end() - 1, g) - offset.begin()) - 1u; };
    const uint32_t n = offset.back(), shift = ctx[0].plan.shift;
    const orc_view& v = *view;
    Frame F;
    F.keys.resize(n); F.order.resize(n);
    for (uint32_t g = 0; g < n; ++g) {
        const uint32_t j = seg(g);
        F.keys[g] = key_of(cl[j].pos_vis + 4 * (size_t)(g - offset[j]), v, cl[j].u, shift).key;
    }
    std::iota(F.order.begin(), F.order.end(), 0u);
    const uint32_t* kp = F.keys.data();
    std::stable_sort(F.order.begin(), F.order.end(), [kp](uint32_t a, uint32_t b) { return kp[a] < kp[b]; });
    uint32_t nv = 0;
    const uint32_t culled = 0xFFFFFFFFu >> shift;
    while (nv < n && F.keys[F.order[nv]] != culled) ++nv;
    F.n_vis = nv;
    *n_vis = nv;
    if (sorted) for (uint32_t e = 0; e < n; ++e) { sorted[2 * e] = F.keys[F.order[e]]; sorted[2 * e + 1] = F.order[e]; }
    auto dist = [&](uint32_t g) {
        const uint32_t j = seg(g);
        float pw[4];
        const float* p = cl[j].pos_vis + 4 * (size_t)(g - offset[j]);
        mat4_point(cl[j].u.transform, p[0], p[1], p[2], pw);
        const float d[3] = {pw[0] - v.world_position[0], pw[1] - v.world_position[1], pw[2] - v.world_position[2]};
        return std::sqrt(dot3(d, d));
    };
    float dmin = 0.0f, dmax = 0.0f;
    if (n >= 2) { dmin = dist(F.order[n - 1]); dmax = dist(F.order[1]); }
    F.splats.resize(nv); F.rank_to_id.resize(nv);
    std::vector<float> dz(nv);
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)nv; ++r) {
        const uint32_t g = F.order[nv - 1 - r], j = seg(g);
        const size_t i = g - offset[j];
        const s4o_cloud& c = cl[j];
        F.rank_to_id[r] = g;
        const float* p = c.pos_vis + 4 * i;
        if (c.kind == 1u) {
            const Rec4 q = project4(ctx[j], tp[j], p, c.sh + 144 * i, c.rot + 8 * i, c.scale_opacity + 4 * i, c.tt + 4 * i, dmin,
                                    dmax, n);
            F.splats[r] = q.sp;
            dz[r] = q.d;
            continue;
        }
        orc_splat& o = F.splats[r];
        const KeyOut kb = key_of(p, v, c.u, 0);
        dz[r] = splat_depth_at(v, kb.pw);
        if (st[j].rasterize_mode == 6u) {   // Velocity: a 3D gaussian is undrawn (centre and opacity only)
            orc_settings s0 = st[j];
            s0.rasterize_mode = 0u; s0.draw_mode = 0u;
            Ctx c0 = ctx[j];
            c0.s = &s0;
            project_one(c0, p, c.sh + 48 * i, c.rot + 4 * i, c.scale_opacity + 4 * i, o);
            const float cx = o.cx, cy = o.cy, op = o.op;
            std::memset(&o, 0, sizeof(o));
            set_bbox_empty(o);
            o.cx = cx; o.cy = cy; o.op = op;
            continue;
        }
        project_one(ctx[j], p, c.sh + 48 * i, c.rot + 4 * i, c.scale_opacity + 4 * i, o);
        if (st[j].rasterize_mode == 1u && n >= 2 && o.xlo <= o.xhi) {   // the Depth colour from the joint range
            float rgb[3];
            depth_to_rgb(dist(g), dmin, dmax, rgb);
            if (!(st[j].draw_mode == 2u && p[3] > 0.5f)) { o.r = rgb[0]; o.g = rgb[1]; o.b = rgb[2]; }
        }
    }
    // each splat's blend: its own entity's (the blend of a 4D record is the 3D one)
    std::vector<orc_settings> sb(st);
    for (orc_settings& s : sb)
        if (s.gaussian_mode == 2u) s.gaussian_mode = 1u;
    std::vector<uint32_t> seg_of(nv);
    for (uint32_t r = 0; r < nv; ++r) {
        seg_of[r] = seg(F.rank_to_id[r]);
        if (records) to_record(F.splats[r], st[seg_of[r]].aabb != 0u, records + 12 * (size_t)r);
        if (rank_to_id) rank_to_id[r] = F.rank_to_id[r];
        if (depths) depths[r] = dz[r];
    }
    const int W = ctx[0].Wi, H = ctx[0].Hi;
    const int TX = (W + TILE - 1) / TILE, TY = (H + TILE - 1) / TILE, NT = TX * TY;
    std::vector<uint64_t> count;
    std::vector<uint32_t> entries;
    bin_tiles(F, TX, TY, count, entries);
    if (n_pairs) *n_pairs = count[NT];
    if (tile_ranges) for (int t = 0; t < NT; ++t) {
        const bool empty = count[t] == count[t + 1];
        tile_ranges[2 * t] = empty ? 0u : (uint32_t)count[t];
        tile_ranges[2 * t + 1] = empty ? 0u : (uint32_t)count[t + 1];
    }
    if (tile_entries) std::memcpy(tile_entries, entries.data(), (size_t)std::min<uint64_t>(count[NT], cap) * 4);
    if (!image) return 0;
#pragma omp parallel for schedule(dynamic, 4)
    for (int t = 0; t < NT; ++t) {   // s4o_frame's walk, each splat by its own entity's coverage rule
        const int tx = t % TX, ty = t / TX;
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
            for (uint64_t e = count[t]; e < count[t + 1]; ++e) {
                const orc_splat& sp = F.splats[entries[e]];
                float a;
                if (!eval_alpha(sp, sb[seg_of[entries[e]]], (float)x + 0.5f, (float)y + 0.5f, &a)) continue;
                if (scene) {
                    const float zs = *reinterpret_cast<const float*>(reinterpret_cast<const char*>(scene) + (uint64_t)y * pitch_bytes + 4u * (uint64_t)x);
                    if (!(dz[entries[e]] >= zs)) continue;
                }
                const float w = a * T;
                cr += w * sp.r; cg += w * sp.g; cb += w * sp.b;
                T = T * (1.0f - a);
                if (T < T_STOP) break;
            }
            float* px = image + 4 * ((size_t)y * W + x);
            px[0] = cr; px[1] = cg; px[2] = cb; px[3] = 1.0f;
        }
    }
    return 0;
}

}  // extern "C"
