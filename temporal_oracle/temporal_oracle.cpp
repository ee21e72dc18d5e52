// temporal_oracle.cpp -- see temporal_oracle.h.  The oracle's translation unit is compiled into this one, so key-gen,
// the sort, binning and the coverage decision below are oracle/'s unchanged; the 4D record and its colours are new.
#include "../oracle/bgs_oracle.cpp"

#include "temporal_oracle.h"

#include "../modes_oracle/modes_oracle.h"

namespace {

// include/bgs.h (bgs_render_4d, 4.): range reduction by ln 2, Taylor to degree 16, times 2^k, rounded to f32
float det_exp(float xf) {
    if (std::isnan(xf)) return xf;
    if (xf < -110.0f) return 0.0f;
    if (xf > 89.0f) return INFINITY;
    const double x = (double)xf;
    const double k = std::rint(x * 1.4426950408889634);
    const double r = x - k * 0.6931471805599453;
    double c[17];
    c[0] = 1.0;
    for (int j = 1; j <= 16; ++j) c[j] = c[j - 1] / (double)j;
    double p = c[16];
    for (int j = 15; j >= 0; --j) p = p * r + c[j];
    const uint64_t bits = (uint64_t)((int)k + 1023) << 52;
    double scale;
    std::memcpy(&scale, &bits, 8);
    return (float)(p * scale);
}

// include/bgs.h (bgs_render_4d, 7.): reduction by 2 pi, Taylor to degree 36, rounded to f32; not finite: NaN
float det_cos(float xf) {
    if (!(std::fabs(xf) < INFINITY)) return std::nanf("");
    const double x = (double)xf;
    const double k = std::rint(x * 0.15915494309189535);
    const double r = x - k * 6.283185307179586;
    const double z = r * r;
    double c[19];
    c[0] = 1.0;
    for (int j = 1; j <= 18; ++j) c[j] = -c[j - 1] / (double)((2 * j - 1) * (2 * j));
    double p = c[18];
    for (int j = 17; j >= 0; --j) p = p * z + c[j];
    return (float)p;
}

struct Cond {
    float c3[6], dm[3], marginal;
    bool mask;
};

// gaussian_4d.wgsl:37-130, matrices [col][row]
Cond condition(float gs, const float* q8, const float* so, const float* tt, float t) {
    Cond g{};
    const float dt = t - tt[0];
    const float sd[4] = {gs * so[0], gs * so[1], gs * so[2], tt[1]};
    const float w = q8[0], x = q8[1], y = q8[2], z = q8[3], wr = q8[4], xr = q8[5], yr = q8[6], zr = q8[7];
    const float Ml[4][4] = {{w, -x, -y, -z}, {x, w, -z, y}, {y, z, w, -x}, {z, -y, x, w}};
    const float Mr[4][4] = {{wr, -xr, -yr, -zr}, {xr, wr, zr, -yr}, {yr, -zr, wr, xr}, {zr, yr, -xr, wr}};
    float R[4][4], M[4][4], S[4][4];
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) R[c][r] = ((Mr[0][r] * Ml[c][0] + Mr[1][r] * Ml[c][1]) + Mr[2][r] * Ml[c][2]) + Mr[3][r] * Ml[c][3];
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) M[c][r] = R[c][r] * sd[c];
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) S[c][r] = ((M[r][0] * M[c][0] + M[r][1] * M[c][1]) + M[r][2] * M[c][2]) + M[r][3] * M[c][3];
    const float cov_t = S[3][3];
    g.marginal = det_exp(((-0.5f * dt) * dt) / cov_t);
    g.mask = g.marginal > 0.05f;
    if (!g.mask) return g;
    const float c12[3] = {S[0][3], S[1][3], S[2][3]};
    auto cond = [&](int c, int r) { return S[c][r] - (c12[c] * c12[r]) / cov_t; };
    g.c3[0] = cond(0, 0); g.c3[1] = cond(0, 1); g.c3[2] = cond(0, 2);
    g.c3[3] = cond(1, 1); g.c3[4] = cond(1, 2); g.c3[5] = cond(2, 2);
    for (int i = 0; i < 3; ++i) g.dm[i] = (c12[i] / cov_t) * dt;
    return g;
}

// helpers.wgsl:8-119 on the conditioned covariance at pw: the OBB or AABB record into o (centre already set)
void geometry(const Ctx& C, const float pw[3], const float c3[6], float cutoff, orc_splat& o) {
    const orc_view& v = *C.v;
    const float W = C.W, H = C.H;
    const float Vrk[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
    float t[4];
    mat4_point(v.view_from_world, pw[0], pw[1], pw[2], t);
    const float fx = v.clip_from_view[0] * W, fy = v.clip_from_view[5] * H;
    const float sz = 1.0f / (t[2] * t[2]);
    const float J00 = fx / t[2], J20 = -(fx * t[0]) * sz;
    const float J11 = -fy / t[2], J21 = (fy * t[1]) * sz;
    float Tm[3][2];
    for (int i = 0; i < 3; ++i) {
        const float v0 = v.view_from_world[i * 4 + 0], v1 = v.view_from_world[i * 4 + 1], v2 = v.view_from_world[i * 4 + 2];
        Tm[i][0] = v0 * J00 + v2 * J20;
        Tm[i][1] = v1 * J11 + v2 * J21;
    }
    float Y[3][2];
    for (int i = 0; i < 3; ++i)
        for (int b = 0; b < 2; ++b) Y[i][b] = (Vrk[i][0] * Tm[0][b] + Vrk[i][1] * Tm[1][b]) + Vrk[i][2] * Tm[2][b];
    const float a = ((Tm[0][0] * Y[0][0] + Tm[1][0] * Y[1][0]) + Tm[2][0] * Y[2][0]) + 0.3f;
    const float b = (Tm[0][1] * Y[0][0] + Tm[1][1] * Y[1][0]) + Tm[2][1] * Y[2][0];
    const float c = ((Tm[0][1] * Y[0][1] + Tm[1][1] * Y[1][1]) + Tm[2][1] * Y[2][1]) + 0.3f;
    const float det = a * c - b * b;
    const float mid = 0.5f * (a + c);
    const float term = std::sqrt(std::fmax(0.0f, mid * mid - det));
    const float l1 = mid + term;
    if (C.s->aabb) {
        const float l2 = std::fmax(mid - term, 0.0f);
        const float Rq = cutoff * std::fmax(std::sqrt(l1), std::sqrt(l2));
        const float dinv = 1.0f / det;
        o.extra[0] = c * dinv; o.extra[1] = -b * dinv; o.extra[2] = a * dinv; o.extra[3] = Rq;
        const float h = 0.5f * Rq;
        set_bbox(o, o.cx, o.cy, h, h, C.Wi, C.Hi);
    } else {
        const float aa = (a - c) * (a - c);
        const float bb = std::sqrt(aa + (4.0f * b) * b);
        const float major = std::sqrt(((a + c) + bb) * 0.5f);
        const float minor = std::sqrt(((a + c) - bb) * 0.5f);
        const float Bx = cutoff * major, By = cutoff * minor;
        const float evx = -b, evy = l1 - a;
        const float el = std::sqrt(evx * evx + evy * evy);
        const float e1x = evx / el, e1y = evy / el;
        const float e2x = e1y, e2y = -e1x;
        o.ux = (2.0f * e1x) / Bx; o.uy = (-2.0f * e1y) / Bx;
        o.vx = (2.0f * e2x) / By; o.vy = (-2.0f * e2y) / By;
        const float hx = 0.5f * (std::fabs(e1x) * Bx + std::fabs(e2x) * By);
        const float hy = 0.5f * (std::fabs(e1y) * Bx + std::fabs(e2y) * By);
        if (o.ux == o.ux && o.uy == o.uy && o.vx == o.vx && o.vy == o.vy) set_bbox(o, o.cx, o.cy, hx, hy, C.Wi, C.Hi);
    }
}

// spherindrical_harmonics.wgsl:11-126 along the camera ray to pw in the model frame, then the sRGB decode
void spherindrical(const Ctx& C, const tor_temporal& tp, const float pw[3], float dt, const float* sh, float rgb[3]) {
    const orc_view& v = *C.v; const orc_uniform& u = *C.u;
    const float dlt[3] = {pw[0] - v.world_position[0], pw[1] - v.world_position[1], pw[2] - v.world_position[2]};
    float dw[3], loc[3], dl[3];
    normalize3(dlt, dw);
    for (int c = 0; c < 3; ++c) {
        const float col[3] = {u.transform[c * 4 + 0], u.transform[c * 4 + 1], u.transform[c * 4 + 2]};
        float bn[3];
        normalize3(col, bn);
        loc[c] = dot3(bn, dw);
    }
    normalize3(loc, dl);
    sh_lookup(sh, dl, rgb);
    const float x = dl[0], y = dl[1], z = dl[2];
    const float xx = x * x, yy = y * y, zz = z * z;
    const float basis[16] = {1.0f, y, z, x, x * y, y * z, (2.0f * zz - xx) - yy, x * z, xx - yy, y * (3.0f * xx - yy),
                             (x * y) * z, y * ((4.0f * zz - xx) - yy), z * ((2.0f * zz - 3.0f * xx) - 3.0f * yy),
                             x * ((4.0f * zz - xx) - yy), z * (xx - yy), x * (xx - 3.0f * yy)};
    const float theta = dt / (tp.time_stop - tp.time_start);
    const float pi = 3.14159274f;
    const float t1 = det_cos((2.0f * pi) * theta), t2 = det_cos((4.0f * pi) * theta);
    for (int c = 0; c < 3; ++c) {
        float s1 = 0.0f, s2 = 0.0f;
        for (int k = 0; k < 16; ++k) {
            s1 += (SHC[k] * basis[k]) * sh[48 + 3 * k + c];
            s2 += (SHC[k] * basis[k]) * sh[96 + 3 * k + c];
        }
        rgb[c] = (rgb[c] + t1 * s1) + t2 * s2;
        if (u.color_space == 0u) rgb[c] = srgb_to_linear(rgb[c]);
    }
}

void flow(const float* clip, const tor_temporal& tp, const float pw[3], const float p0[3], float rgb[3]) {
    float c[4], cp[4];
    mat4_point(clip, pw[0], pw[1], pw[2], c);
    mat4_point(tp.prev_clip_from_world, p0[0], p0[1], p0[2], cp);
    const float mvx = (c[0] / c[3] - cp[0] / cp[3]) * 0.5f;
    const float mvy = (c[1] / c[3] - cp[1] / cp[3]) * -0.5f;
    const float fx = mvx / tp.delta_time, fy = mvy / tp.delta_time;
    const float radius = std::sqrt(fx * fx + fy * fy);
    float angle;
    mo_atan2(1, &fy, &fx, &angle);
    if (angle < 0.0f) angle = angle + 6.28318530718f;
    const float s = std::fmin(std::fmax(radius, 0.0f), 1.0f), one = 1.0f;
    mo_hsv_to_rgb(1, &angle, &s, &one, rgb);
}

struct Rec4 {
    orc_splat sp;
    float d;   // the depth-test depth
};

// include/bgs.h (bgs_render_4d) for one gaussian; dmin / dmax: the Depth colour's range
Rec4 project4(const Ctx& C, const tor_temporal& tp, const float* p4, const float* sh, const float* q8, const float* so,
              const float* tt, float dmin, float dmax, uint32_t n) {
    const orc_view& v = *C.v; const orc_uniform& u = *C.u; const orc_settings& s = *C.s;
    Rec4 out;
    orc_splat& o = out.sp;
    std::memset(&o, 0, sizeof(o));
    set_bbox_empty(o);
    const KeyOut k = key_of(p4, v, u, 0);
    const float hw = 0.5f * C.W, hh = 0.5f * C.H;
    o.cx = k.ndc[0] * hw + hw;
    o.cy = hh - k.ndc[1] * hh;
    const float opacity = so[3];
    o.op = opacity * u.global_opacity;
    float pd[3] = {k.pw[0], k.pw[1], k.pw[2]};
    auto depth_of = [&](const float pw[3]) {
        float c[4];
        mat4_point(v.clip_from_world, pw[0], pw[1], pw[2], c);
        const float den = c[3] + 0.000000001f;
        return (c[2] / den) / (c[3] / den);
    };
    if (k.visible && !(s.draw_mode == 1u && p4[3] < 0.5f)) {
        float cutoff = 3.0f;
        if (s.opacity_adaptive_radius) {
            const float a = 9.0f + 2.0f * det_ln(opacity);
            cutoff = std::sqrt(a > 0.000001f ? a : 0.000001f);
        }
        const Cond g = condition(u.global_scale, q8, so, tt, u.time);
        if (g.mask) {
            const float moved[3] = {p4[0] + g.dm[0], p4[1] + g.dm[1], p4[2] + g.dm[2]};
            const KeyOut km = key_of(moved, v, u, 0);
            if (km.visible) {
                o.cx = km.ndc[0] * hw + hw;
                o.cy = hh - km.ndc[1] * hh;
                float op = opacity * g.marginal;
                geometry(C, km.pw, g.c3, cutoff, o);
                float rgb[3] = {0.0f, 0.0f, 0.0f};
                const uint32_t mode = s.rasterize_mode;
                if (mode == 0u || mode == 4u) {
                    spherindrical(C, tp, km.pw, u.time - tt[0], sh, rgb);
                    if (mode == 4u) {
                        float h[3];
                        mo_class_colour(1, rgb, &p4[3], tp.num_classes, h);
                        rgb[0] = h[0]; rgb[1] = h[1]; rgb[2] = h[2];
                    }
                } else if (mode == 1u) {
                    if (n >= 2) {
                        const float d[3] = {km.pw[0] - v.world_position[0], km.pw[1] - v.world_position[1], km.pw[2] - v.world_position[2]};
                        depth_to_rgb(std::sqrt(dot3(d, d)), dmin, dmax, rgb);
                    }
                } else if (mode == 3u) {
                    for (int c = 0; c < 3; ++c) rgb[c] = (km.pw[c] - u.aabb_min[c]) / (u.aabb_max[c] - u.aabb_min[c]);
                } else if (mode == 5u) {
                    flow(v.clip_from_world, tp, km.pw, k.pw, rgb);
                } else {
                    const Cond f = condition(u.global_scale, q8, so, tt, u.time + 1.0e-3f);
                    float vel[3];
                    for (int i = 0; i < 3; ++i) vel[i] = ((f.mask ? f.dm[i] : 0.0f) - g.dm[i]) / 1.0e-3f;
                    const float len = std::sqrt((vel[0] * vel[0] + vel[1] * vel[1]) + vel[2] * vel[2]);
                    const float scaled = std::fmin(std::fmax((len - 1.0f) / (2.0f - 1.0f), 0.0f), 1.0f);
                    if (scaled < 1.0e-2f) op = 0.0f;
                    else for (int i = 0; i < 3; ++i) rgb[i] = (0.5f * (vel[i] / len + 1.0f)) * scaled;
                }
                o.r = rgb[0]; o.g = rgb[1]; o.b = rgb[2];
                o.op = op * u.global_opacity;
                if (s.draw_mode == 2u && p4[3] > 0.5f) { o.r = 0.3f; o.g = 1.0f; o.b = 0.1f; o.op = 1.0f; }
                pd[0] = km.pw[0]; pd[1] = km.pw[1]; pd[2] = km.pw[2];
            }
        }
    }
    out.d = depth_of(pd);
    return out;
}

void to_record(const orc_splat& o, bool aabb, float* r) {
    r[0] = o.cx; r[1] = o.cy;
    const float* uv = aabb ? o.extra : &o.ux;
    r[2] = uv[0]; r[3] = uv[1]; r[4] = uv[2]; r[5] = uv[3];
    const uint32_t bx = (uint32_t)o.xlo | ((uint32_t)o.xhi << 16), by = (uint32_t)o.ylo | ((uint32_t)o.yhi << 16);
    std::memcpy(&r[6], &bx, 4); std::memcpy(&r[7], &by, 4);
    r[8] = o.r; r[9] = o.g; r[10] = o.b; r[11] = o.op;
}

}  // namespace

extern "C" {

void tor_exp(uint32_t n, const float* x, float* out) { for (uint32_t i = 0; i < n; ++i) out[i] = det_exp(x[i]); }
void tor_cos(uint32_t n, const float* x, float* out) { for (uint32_t i = 0; i < n; ++i) out[i] = det_cos(x[i]); }

void tor_condition(uint32_t n, const float* rot8, const float* so, const float* tt, float gs, float t, float* cov6,
                   float* dm, float* marginal, uint8_t* mask) {
    for (uint32_t i = 0; i < n; ++i) {
        const Cond g = condition(gs, rot8 + 8 * (size_t)i, so + 4 * (size_t)i, tt + 4 * (size_t)i, t);
        for (int k = 0; k < 6; ++k) cov6[6 * (size_t)i + k] = g.c3[k];
        for (int k = 0; k < 3; ++k) dm[3 * (size_t)i + k] = g.dm[k];
        marginal[i] = g.marginal;
        mask[i] = g.mask ? 1 : 0;
    }
}

int tor_frame(uint32_t n, const float* pos, const float* sh, const float* rot8, const float* so, const float* tt,
              const orc_view* view, const orc_uniform* u, const orc_settings* s, const tor_temporal* tp, const float* scene,
              uint64_t pitch_bytes, uint32_t* n_vis, float* records, uint32_t* rank_to_id, float* depths, float* image,
              int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s) || !tp) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    // key-gen and the sort: a 3D cloud's, on the base positions
    Frame F;
    F.keys.resize(n); F.order.resize(n);
    for (uint32_t i = 0; i < n; ++i) F.keys[i] = key_of(pos + 4 * (size_t)i, *view, *u, C.plan.shift).key;
    std::iota(F.order.begin(), F.order.end(), 0u);
    const uint32_t* kp = F.keys.data();
    std::stable_sort(F.order.begin(), F.order.end(), [kp](uint32_t a, uint32_t b) { return kp[a] < kp[b]; });
    uint32_t nv = 0;
    const uint32_t culled = 0xFFFFFFFFu >> C.plan.shift;
    while (nv < n && F.keys[F.order[nv]] != culled) ++nv;
    F.n_vis = nv;
    *n_vis = nv;
    if (!records && !image && !depths && !rank_to_id) return 0;
    float dmin = 0.0f, dmax = 0.0f;
    if (n >= 2) {   // gaussian.wgsl:329-349: sorted[N-1] and sorted[1], base positions
        auto dist = [&](uint32_t id) {
            float pw[4]; const float* p = pos + 4 * (size_t)id;
            mat4_point(u->transform, p[0], p[1], p[2], pw);
            const float d[3] = {pw[0] - view->world_position[0], pw[1] - view->world_position[1], pw[2] - view->world_position[2]};
            return std::sqrt(dot3(d, d));
        };
        dmin = dist(F.order[n - 1]); dmax = dist(F.order[1]);
    }
    F.splats.resize(nv); F.rank_to_id.resize(nv);
    std::vector<float> dz(nv);
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)nv; ++r) {
        const size_t id = F.order[nv - 1 - r];
        F.rank_to_id[r] = (uint32_t)id;
        const Rec4 q = project4(C, *tp, pos + 4 * id, sh + 144 * id, rot8 + 8 * id, so + 4 * id, tt + 4 * id, dmin, dmax, n);
        F.splats[r] = q.sp;
        dz[r] = q.d;
    }
    for (uint32_t r = 0; r < nv; ++r) {
        if (records) to_record(F.splats[r], s->aabb != 0u, records + 12 * (size_t)r);
        if (rank_to_id) rank_to_id[r] = F.rank_to_id[r];
        if (depths) depths[r] = dz[r];
    }
    if (!image) return 0;
    orc_settings s3 = *s;
    s3.gaussian_mode = 1u;   // the blend of a 4D record is the 3D one
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
                if (!eval_alpha(sp, s3, (float)x + 0.5f, (float)y + 0.5f, &a)) continue;
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
