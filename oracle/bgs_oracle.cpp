// bgs_oracle.cpp -- CPU ORACLE (test infrastructure; see bgs_oracle.h for the rules).
//
// A restatement, in plain C++ with a fixed FP policy, of the reference's forward splat path
// (mosure/bevy_gaussian_splatting @ d6a4432).  Each function cites the reference file:line it
// follows.  Nothing here is copied from the reference: the WGSL is re-expressed as scalar
// maths in (row, col) notation with an explicit evaluation order.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fopenmp -shared -fPIC (see oracle/Makefile).
// -ffp-contract=off is REQUIRED: every a*b+c below is a rounded multiply then a rounded add.
//
// Conventions: matrices arrive column-major as Bevy/WGSL store them: m[c*4 + r].
// min()/max() on floats follow IEEE minNum/maxNum (fmin/fmax: a NaN operand is ignored), the same as the
// CUDA fminf/fmaxf the kernels use; WGSL leaves the NaN case implementation-defined.
#include "bgs_oracle.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#include <parallel/algorithm>
#endif

namespace {

constexpr int TILE = 16;
constexpr float T_STOP = 1.0e-4f;   // tile_mode: a pixel stops once its transmittance < T_STOP

inline uint32_t f2u(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline float u2f(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

// M * (x,y,z,1), summed ((m0*x + m1*y) + m2*z) + m3   (policy: SURVEY.md Appendix A.2)
inline void mat4_point(const float* m, float x, float y, float z, float out[4]) {
    for (int r = 0; r < 4; ++r) out[r] = ((m[0 + r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r];
}
// M * (x,y,z,0)
inline void mat4_dir(const float* m, float x, float y, float z, float out[4]) {
    for (int r = 0; r < 4; ++r) out[r] = (m[0 + r] * x + m[4 + r] * y) + m[8 + r] * z;
}

// ---- src/render/mod.rs:715-760 (ShaderDefines::for_radix_depth_bits, radix_initial_parity)
struct PassPlan { uint32_t places, shift, parity; };
inline PassPlan pass_plan(uint32_t bits) {
    PassPlan p;
    p.places = bits / 8u;       // radix_bits_per_digit = 8
    p.shift = 32u - bits;       // radix_key_shift
    p.parity = p.places % 2u;   // radix_initial_parity
    return p;
}

// ---- src/sort/radix.wgsl:86-101 + src/render/transform.wgsl:5-14
struct KeyOut { uint32_t key; bool visible; float pw[3]; float ndc[4]; float d2; };
inline KeyOut key_of(const float* p, const orc_view& v, const orc_uniform& u, uint32_t shift) {
    KeyOut k;
    float pw4[4];
    mat4_point(u.transform, p[0], p[1], p[2], pw4);
    k.pw[0] = pw4[0]; k.pw[1] = pw4[1]; k.pw[2] = pw4[2];
    float c[4];
    mat4_point(v.clip_from_world, k.pw[0], k.pw[1], k.pw[2], c);   // unjittered_clip_from_world
    const float den = c[3] + 0.000000001f;
    for (int i = 0; i < 4; ++i) k.ndc[i] = c[i] / den;
    k.visible = std::fabs(k.ndc[0]) < 1.1f && std::fabs(k.ndc[1]) < 1.1f &&
                std::fabs(k.ndc[2] - 0.5f) < 0.5f;
    const float dx = k.pw[0] - v.world_position[0];
    const float dy = k.pw[1] - v.world_position[1];
    const float dz = k.pw[2] - v.world_position[2];
    k.d2 = (dx * dx + dy * dy) + dz * dz;
    uint32_t key = 0xFFFFFFFFu;
    if (k.visible) key = 0xFFFFFFFFu - f2u(k.d2);
    k.key = key >> shift;
    return k;
}

// ---- fixed-series natural log (policy item; replaces WGSL log() in gaussian.wgsl:229).
// double precision: x = m * 2^e, m in [sqrt(1/2), sqrt(2)); s = (m-1)/(m+1);
// ln x = e*ln2 + 2*(s + s^3/3 + ... + s^23/23), Horner in s^2, then rounded to f32.
inline float det_ln(float xf) {
    if (xf != xf) return xf;
    if (xf < 0.0f) return std::numeric_limits<float>::quiet_NaN();
    if (xf == 0.0f) return -std::numeric_limits<float>::infinity();
    if (xf == std::numeric_limits<float>::infinity()) return xf;
    double x = (double)xf;   // exact; every finite f32 (incl. subnormals) is a normal f64
    uint64_t bits; std::memcpy(&bits, &x, 8);
    int e = (int)((bits >> 52) & 0x7FF) - 1023;
    bits = (bits & 0x000FFFFFFFFFFFFFull) | 0x3FF0000000000000ull;
    double m; std::memcpy(&m, &bits, 8);           // m in [1,2)
    if (m > 1.4142135623730951) { m = m * 0.5; e += 1; }
    const double s = (m - 1.0) / (m + 1.0);
    const double z = s * s;
    double p = 1.0 / 23.0;
    p = p * z + 1.0 / 21.0;
    p = p * z + 1.0 / 19.0;
    p = p * z + 1.0 / 17.0;
    p = p * z + 1.0 / 15.0;
    p = p * z + 1.0 / 13.0;
    p = p * z + 1.0 / 11.0;
    p = p * z + 1.0 / 9.0;
    p = p * z + 1.0 / 7.0;
    p = p * z + 1.0 / 5.0;
    p = p * z + 1.0 / 3.0;
    p = p * z + 1.0;
    const double r = (double)e * 0.6931471805599453 + 2.0 * (s * p);
    return (float)r;
}

// ---- software binary16 <-> binary32 (half 2.7 `f16::from_f32` = IEEE RNE; f16.rs:244-263)
inline uint16_t f32_to_f16(float f) {
    const uint32_t x = f2u(f);
    const uint32_t sign = (x >> 16) & 0x8000u;
    const uint32_t ax = x & 0x7FFFFFFFu;
    if (ax >= 0x7F800000u) return (uint16_t)(sign | (ax > 0x7F800000u ? 0x7E00u : 0x7C00u));
    if (ax >= 0x477FF000u) return (uint16_t)(sign | 0x7C00u);     // rounds to inf (>= 65520)
    if (ax < 0x33000001u) return (uint16_t)sign;                  // <= 2^-25 rounds to zero
    int e = (int)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7FFFFFu) | 0x800000u;
    int shift;
    uint32_t he;
    if (e < -14) { shift = 13 + (-14 - e); he = 0; }             // subnormal half
    else { shift = 13; he = (uint32_t)(e + 15); }
    uint32_t hm = m >> shift;
    const uint32_t rem = m & ((1u << shift) - 1u);
    const uint32_t half = 1u << (shift - 1);
    if (rem > half || (rem == half && (hm & 1u))) hm += 1u;
    uint32_t h;
    if (he == 0) h = hm;                 // hm may carry into the exponent field: that is correct
    else h = ((he - 1u) << 10) + hm;     // hm includes the implicit bit (0x400), carries propagate
    return (uint16_t)(sign | h);
}
inline float f16_to_f32(uint16_t h) {
    const uint32_t sign = ((uint32_t)h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1Fu;
    uint32_t m = h & 0x3FFu;
    if (e == 0) {
        if (m == 0) return u2f(sign);
        int sh = 0;
        while (!(m & 0x400u)) { m <<= 1; ++sh; }
        m &= 0x3FFu;
        return u2f(sign | ((uint32_t)(127 - 15 + 1 - sh) << 23) | (m << 13));
    }
    if (e == 31) return u2f(sign | 0x7F800000u | (m << 13));
    return u2f(sign | ((e + 127 - 15) << 23) | (m << 13));
}

// ---- src/material/spherical_harmonics.wgsl:3-20 (constants, signed)
const float SHC[16] = {
    0.28209479177387814f, -0.4886025119029199f, 0.4886025119029199f, -0.4886025119029199f,
    1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
    0.5462742152960396f, -0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
    0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

// ---- spherical_harmonics.wgsl:34-68: 0.5 + sum_k shc[k] * basis_k(dir) * C_k
inline void sh_lookup(const float* sh, const float d[3], float rgb[3]) {
    const float x = d[0], y = d[1], z = d[2];
    const float xx = x * x, yy = y * y, zz = z * z;
    float basis[16];
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
    for (int c = 0; c < 3; ++c) {
        float acc = 0.5f;
        for (int k = 0; k < 16; ++k) acc += (SHC[k] * sh[3 * k + c]) * basis[k];
        rgb[c] = acc;
    }
}
// ---- spherical_harmonics.wgsl:22-32 (no clamp either side)
inline float srgb_to_linear(float v) {
    if (v <= 0.04045f) return v / 12.92f;
    return std::pow((v + 0.055f) / 1.055f, 2.4f);
}

inline void normalize3(const float a[3], float out[3]) {
    const float l = std::sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]);
    out[0] = a[0] / l; out[1] = a[1] / l; out[2] = a[2] / l;
}

// ---- helpers.wgsl:137-158: entries of the matrix the WGSL constructor denotes, as (row, col)
inline void rotation_rows(const float q[4], float R[3][3]) {
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    R[0][0] = 1.0f - 2.0f * (y * y + z * z);
    R[1][0] = 2.0f * (x * y - r * z);
    R[2][0] = 2.0f * (x * z + r * y);
    R[0][1] = 2.0f * (x * y + r * z);
    R[1][1] = 1.0f - 2.0f * (x * x + z * z);
    R[2][1] = 2.0f * (y * z - r * x);
    R[0][2] = 2.0f * (x * z - r * y);
    R[1][2] = 2.0f * (y * z + r * x);
    R[2][2] = 1.0f - 2.0f * (x * x + y * y);
}

inline float dot3(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

struct Ctx {
    const orc_view* v; const orc_uniform* u; const orc_settings* s;
    float W, H; int Wi, Hi;
    PassPlan plan;
};

inline void set_bbox_empty(orc_splat& o) { o.xlo = 1; o.xhi = 0; o.ylo = 1; o.yhi = 0; }

// conservative pixel bbox for |fx - cx| <= hx, |fy - cy| <= hy   (a7; this repo's rule)
inline void set_bbox(orc_splat& o, float cx, float cy, float hx, float hy, int Wi, int Hi) {
    set_bbox_empty(o);
    if (!(hx >= 0.0f) || !(hy >= 0.0f) || !(cx == cx) || !(cy == cy)) return;   // NaN => empty
    const float sx = hx * 1.0e-3f + 1.0e-2f, sy = hy * 1.0e-3f + 1.0e-2f;       // slack
    float x0 = std::ceil((cx - hx) - (0.5f + sx));
    float x1 = std::floor((cx + hx) - (0.5f - sx));
    float y0 = std::ceil((cy - hy) - (0.5f + sy));
    float y1 = std::floor((cy + hy) - (0.5f - sy));
    if (!(x0 <= x1) || !(y0 <= y1)) return;
    x0 = std::fmax(x0, 0.0f); y0 = std::fmax(y0, 0.0f);
    x1 = std::fmin(x1, (float)(Wi - 1)); y1 = std::fmin(y1, (float)(Hi - 1));
    if (!(x0 <= x1) || !(y0 <= y1)) return;
    o.xlo = (int)x0; o.xhi = (int)x1; o.ylo = (int)y0; o.yhi = (int)y1;
}

// ---- gaussian.wgsl:185-436 for one gaussian already known visible (key != culled)
void project_one(const Ctx& C, const float* p4, const float* sh, const float* q, const float* so,
                 orc_splat& o) {
    const orc_view& v = *C.v; const orc_uniform& u = *C.u; const orc_settings& s = *C.s;
    std::memset(&o, 0, sizeof(o));
    set_bbox_empty(o);
    const KeyOut k = key_of(p4, v, u, 0);
    // draw modes: gaussian.wgsl:204-206 (DRAW_SELECTED) -- visibility < 0.5 discards
    if (!k.visible) return;
    if (s.draw_mode == 1u && p4[3] < 0.5f) return;
    const float W = C.W, H = C.H;
    const float opacity = so[3];
    float cutoff = 3.0f;
    if (s.opacity_adaptive_radius) {                        // gaussian.wgsl:228-232
        const float a = 9.0f + 2.0f * det_ln(opacity);
        cutoff = std::sqrt(a > 0.000001f ? a : 0.000001f);
    }
    float A[3][3];                                          // model 3x3, (row, col)
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) A[r][c] = u.transform[c * 4 + r];
    float Rm[3][3];
    rotation_rows(q, Rm);
    const float sc[3] = {so[0] * u.global_scale, so[1] * u.global_scale, so[2] * u.global_scale};
    // quad centre in pixels: ndc -> px   (x right, y down)
    const float hw = 0.5f * W, hh = 0.5f * H;
    const float cx = k.ndc[0] * hw + hw;
    const float cy = hh - k.ndc[1] * hh;
    o.cx = cx; o.cy = cy;
    o.op = opacity * u.global_opacity;

    if (s.gaussian_mode == 1u) {
        // ---- gaussian_3d.wgsl:49-72  Sigma = M^T M, M = S R; TS = T Sigma T^T
        float M[3][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) M[i][j] = sc[i] * Rm[i][j];
        float Sg[3][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
            Sg[i][j] = (M[0][i] * M[0][j] + M[1][i] * M[1][j]) + M[2][i] * M[2][j];
        float X[3][3], TS[3][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
            X[i][j] = (A[i][0] * Sg[0][j] + A[i][1] * Sg[1][j]) + A[i][2] * Sg[2][j];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
            TS[i][j] = (X[i][0] * A[j][0] + X[i][1] * A[j][1]) + X[i][2] * A[j][2];
        // cov3d = (TS[0][0], TS[0][1], TS[0][2], TS[1][1], TS[1][2], TS[2][2]) in WGSL [col][row]
        float c3[6] = {TS[0][0], TS[1][0], TS[2][0], TS[1][1], TS[2][1], TS[2][2]};
        if (s.reserved & 1u) {
            // PRECOMPUTE_COVARIANCE_3D (gaussian_3d.wgsl:78-79, planar.wgsl:133-152): get_cov3d(index) goes straight into
            // cov2d -- no global_scale, no model transform.  The caller hands the decoded Covariance3dOpacityPacked128 in
            // the plane slots it occupies: rotation = (c0, c1, c2, c3), scale_opacity = (c4, c5, opacity, opacity).
            c3[0] = q[0]; c3[1] = q[1]; c3[2] = q[2]; c3[3] = q[3]; c3[4] = so[0]; c3[5] = so[1];
        }
        float Vrk[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
        // ---- helpers.wgsl:8-47
        float t[4];
        mat4_point(v.view_from_world, k.pw[0], k.pw[1], k.pw[2], t);
        const float fx = v.clip_from_view[0] * W, fy = v.clip_from_view[5] * H;
        const float sz = 1.0f / (t[2] * t[2]);
        const float J00 = fx / t[2], J20 = -(fx * t[0]) * sz;
        const float J11 = -fy / t[2], J21 = (fy * t[1]) * sz;
        float Tm[3][2];   // T = W * J, W = transpose(view3x3): T[i][a] = sum_k V3[k][i] J[k][a]
        for (int i = 0; i < 3; ++i) {
            const float v0 = v.view_from_world[i * 4 + 0], v1 = v.view_from_world[i * 4 + 1],
                        v2 = v.view_from_world[i * 4 + 2];   // V3[k][i] = column i, row k
            Tm[i][0] = v0 * J00 + v2 * J20;
            Tm[i][1] = v1 * J11 + v2 * J21;
        }
        float Y[3][2];
        for (int i = 0; i < 3; ++i) for (int b = 0; b < 2; ++b)
            Y[i][b] = (Vrk[i][0] * Tm[0][b] + Vrk[i][1] * Tm[1][b]) + Vrk[i][2] * Tm[2][b];
        const float cov00 = ((Tm[0][0] * Y[0][0] + Tm[1][0] * Y[1][0]) + Tm[2][0] * Y[2][0]) + 0.3f;
        const float cov01 = (Tm[0][1] * Y[0][0] + Tm[1][1] * Y[1][0]) + Tm[2][1] * Y[2][0];
        const float cov11 = ((Tm[0][1] * Y[0][1] + Tm[1][1] * Y[1][1]) + Tm[2][1] * Y[2][1]) + 0.3f;
        const float a = cov00, b = cov01, c = cov11;
        // ---- helpers.wgsl:49-67
        const float det = a * c - b * b;
        const float mid = 0.5f * (a + c);
        const float disc = std::fmax(0.0f, mid * mid - det);
        const float term = std::sqrt(disc);
        const float l1 = mid + term;
        if (s.aabb) {
            // ---- helpers.wgsl:69-79, gaussian.wgsl:299-309: square of half-side cutoff*sqrt(l1)
            const float l2 = std::fmax(mid - term, 0.0f);
            const float Rq = cutoff * std::fmax(std::sqrt(l1), std::sqrt(l2));
            const float dinv = 1.0f / det;
            o.extra[0] = c * dinv; o.extra[1] = -b * dinv; o.extra[2] = a * dinv; o.extra[3] = Rq;
            const float h = 0.5f * Rq;
            set_bbox(o, cx, cy, h, h, C.Wi, C.Hi);
        } else {
            // ---- helpers.wgsl:81-119
            const float aa = (a - c) * (a - c);
            const float bb = std::sqrt(aa + (4.0f * b) * b);
            const float major = std::sqrt(((a + c) + bb) * 0.5f);
            const float minor = std::sqrt(((a + c) - bb) * 0.5f);
            const float Bx = cutoff * major, By = cutoff * minor;
            const float evx = -b, evy = l1 - a;
            const float el = std::sqrt(evx * evx + evy * evy);
            const float e1x = evx / el, e1y = evy / el;      // NaN when both components are 0
            const float e2x = e1y, e2y = -e1x;
            // pixel offset (dx right, dy down) -> quad uv: d = (2dx, -2dy); u = dot(d,e1)/B.x
            o.ux = (2.0f * e1x) / Bx; o.uy = (-2.0f * e1y) / Bx;
            o.vx = (2.0f * e2x) / By; o.vy = (-2.0f * e2y) / By;
            const float hx = 0.5f * (std::fabs(e1x) * Bx + std::fabs(e2x) * By);
            const float hy = 0.5f * (std::fabs(e1y) * Bx + std::fabs(e2y) * By);
            if (o.ux == o.ux && o.uy == o.uy && o.vx == o.vx && o.vy == o.vy)
                set_bbox(o, cx, cy, hx, hy, C.Wi, C.Hi);
        }
    } else {
        // ---- gaussian_2d.wgsl:77-132 (surfel) + :49-75 (quad)
        float L[3][2];   // first two columns of A * R_std * S, R_std = transpose(Rm)
        for (int j = 0; j < 2; ++j) {
            const float rc[3] = {Rm[j][0] * sc[j], Rm[j][1] * sc[j], Rm[j][2] * sc[j]};
            for (int i = 0; i < 3; ++i) L[i][j] = (A[i][0] * rc[0] + A[i][1] * rc[1]) + A[i][2] * rc[2];
        }
        float G[3][4];   // G[j] = clip_from_world * column j of world_from_local
        mat4_dir(v.clip_from_world, L[0][0], L[1][0], L[2][0], G[0]);
        mat4_dir(v.clip_from_world, L[0][1], L[1][1], L[2][1], G[1]);
        mat4_point(v.clip_from_world, k.pw[0], k.pw[1], k.pw[2], G[2]);
        const float fxk = v.clip_from_view[0] * W / 2.0f, fyk = v.clip_from_view[5] * H / 2.0f;
        const float cxk = (W - 1.0f) / 2.0f, cyk = (H - 1.0f) / 2.0f;   // helpers.wgsl:122-135
        float T0[3], T1[3], T2[3];
        for (int j = 0; j < 3; ++j) {
            T0[j] = fxk * G[j][0] + cxk * G[j][3];
            T1[j] = fyk * G[j][1] + cyk * G[j][3];
            T2[j] = G[j][3];
        }
        const float c2 = cutoff * cutoff;
        const float test[3] = {c2, c2, -1.0f};
        const float tt[3] = {test[0] * T2[0], test[1] * T2[1], test[2] * T2[2]};
        const float d = dot3(tt, T2);
        float Rq = 0.0f, mean[2] = {0.0f, 0.0f};
        bool ok = !(std::fabs(d) < 1.0e-4f);
        if (ok) {
            const float inv = 1.0f / d;
            const float f[3] = {inv * test[0], inv * test[1], inv * test[2]};
            const float t02[3] = {T0[0] * T2[0], T0[1] * T2[1], T0[2] * T2[2]};
            const float t12[3] = {T1[0] * T2[0], T1[1] * T2[1], T1[2] * T2[2]};
            mean[0] = dot3(f, t02); mean[1] = dot3(f, t12);
            const float f0[3] = {f[0] * T0[0], f[1] * T0[1], f[2] * T0[2]};
            const float f1[3] = {f[0] * T1[0], f[1] * T1[1], f[2] * T1[2]};
            const float ex = mean[0] * mean[0] - dot3(f0, T0);
            const float ey = mean[1] * mean[1] - dot3(f1, T1);
            if (ex < 1.0e-4f || ey < 1.0e-4f) ok = false;   // NaN extents fall through (NaN quad)
            else Rq = std::fmax(std::fmax(std::sqrt(ex), std::sqrt(ey)), cutoff * 0.707106f);
        }
        if (ok) {
            o.extra[3] = Rq; o.extra[4] = mean[0]; o.extra[5] = mean[1]; o.extra[6] = W / H;
            for (int j = 0; j < 3; ++j) { o.extra[7 + j] = T0[j]; o.extra[10 + j] = T1[j]; o.extra[13 + j] = T2[j]; }
            o.ux = 2.0f / Rq; o.uy = 0.0f; o.vx = 0.0f; o.vy = -2.0f / Rq;   // OBB branch: e1=(1,0), e2=(0,1)
            const float h = 0.5f * Rq;
            if (Rq == Rq) set_bbox(o, cx, cy, h, h, C.Wi, C.Hi);
        }
    }

    // ---- colour source
    float rgb[3] = {0.0f, 0.0f, 0.0f};
    if (s.rasterize_mode == 0u) {
        // gaussian.wgsl:166-183,406-416 + planar.wgsl:91-106
        const float dlt[3] = {k.pw[0] - v.world_position[0], k.pw[1] - v.world_position[1],
                              k.pw[2] - v.world_position[2]};
        float dw[3]; normalize3(dlt, dw);
        float loc[3];
        for (int c = 0; c < 3; ++c) {
            const float col[3] = {A[0][c], A[1][c], A[2][c]};
            float bn[3]; normalize3(col, bn);
            loc[c] = dot3(bn, dw);
        }
        float dl[3]; normalize3(loc, dl);
        sh_lookup(sh, dl, rgb);
        if (u.color_space == 0u) for (int c = 0; c < 3; ++c) rgb[c] = srgb_to_linear(rgb[c]);
    } else if (s.rasterize_mode == 2u) {
        // gaussian.wgsl:350-368: L = T*S*R; n = normalize(view_from_world * (L[2], 0)); 0.5(n+1)
        float SR[3];   // column 2 of S*R = (sc_i * Rm[i][2])
        for (int i = 0; i < 3; ++i) SR[i] = sc[i] * Rm[i][2];
        float Ln[3];
        for (int i = 0; i < 3; ++i) Ln[i] = (A[i][0] * SR[0] + A[i][1] * SR[1]) + A[i][2] * SR[2];
        float wn[4];
        mat4_dir(v.view_from_world, Ln[0], Ln[1], Ln[2], wn);
        const float l = std::sqrt(((wn[0] * wn[0] + wn[1] * wn[1]) + wn[2] * wn[2]) + wn[3] * wn[3]);
        for (int c = 0; c < 3; ++c) rgb[c] = 0.5f * (wn[c] / l + 1.0f);
    }
    else if (s.rasterize_mode == 3u) {
        // gaussian.wgsl:375-376 RASTERIZE_POSITION: (transformed_position - min) / (max - min); min/max are the
        // entity Aabb's (cloud-space) corners while the position is the world-space one -- kept literal
        for (int c = 0; c < 3; ++c) rgb[c] = (k.pw[c] - u.aabb_min[c]) / (u.aabb_max[c] - u.aabb_min[c]);
    }
    // rasterize_mode == 1 (Depth) is filled by the caller: it needs the sorted order.
    o.r = rgb[0]; o.g = rgb[1]; o.b = rgb[2];
    if (s.draw_mode == 2u && p4[3] > 0.5f) {   // gaussian.wgsl:423-427 HIGHLIGHT_SELECTED
        o.r = 0.3f; o.g = 1.0f; o.b = 0.1f; o.op = 1.0f;
    }
}

// ---- material/depth.wgsl:3-11
inline void depth_to_rgb(float depth, float dmin, float dmax, float rgb[3]) {
    float nd = (depth - dmin) / (dmax - dmin);
    nd = std::fmin(std::fmax(nd, 0.0f), 1.0f);
    auto smooth = [](float e0, float e1, float x) {
        float t = (x - e0) / (e1 - e0);
        t = std::fmin(std::fmax(t, 0.0f), 1.0f);
        return t * t * (3.0f - 2.0f * t);
    };
    rgb[0] = smooth(0.5f, 1.0f, nd);
    rgb[1] = 1.0f - std::fabs(nd - 0.5f) * 2.0f;
    rgb[2] = 1.0f - smooth(0.0f, 0.5f, nd);
}

// ---- fs_main (gaussian.wgsl:439-505) at pixel centre (fx, fy): the quantities the coverage decision turns on.
// `fused` = false computes u, v with a separately rounded multiply and add (what a kernel without the explicit fma
// would do); the decision is then `covered`, and `power` is filled only for covered pixels.
struct Decision { float u, v, mx, my, Rq, power; bool covered; };
inline Decision decide(const orc_splat& sp, const orc_settings& s, float fx, float fy, bool fused = true) {
    Decision d{0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, false};
    const float dx = fx - sp.cx, dy = fy - sp.cy;
    float power;
    if (!s.aabb) {
        // USE_OBB: uv from the quad, power = -|uv|^2 / (2/9)
        d.u = fused ? std::fmaf(sp.uy, dy, sp.ux * dx) : sp.ux * dx + sp.uy * dy;
        d.v = fused ? std::fmaf(sp.vy, dy, sp.vx * dx) : sp.vx * dx + sp.vy * dy;
        const float uu = d.u, vv = d.v;
        if (!(std::fabs(uu) <= 1.0f && std::fabs(vv) <= 1.0f)) return d;
        const float qd = std::fmaf(vv, vv, uu * uu);
        power = -4.5f * qd;
    } else {
        const float mx = dx + dx, my = -(dy + dy);      // quad-space offset in half-pixels (y up)
        const float Rq = sp.extra[3];
        d.mx = mx; d.my = my; d.Rq = Rq;
        if (!(std::fabs(mx) <= Rq && std::fabs(my) <= Rq)) return d;
        if (s.gaussian_mode == 1u) {
            const float ddx = -mx, ddy = -my;            // gaussian.wgsl:459-462
            const float t1 = (sp.extra[0] * ddx) * ddx, t2 = (sp.extra[2] * ddy) * ddy;
            power = -0.5f * (t1 + t2) + (sp.extra[1] * ddx) * ddy;
        } else {
            // gaussian.wgsl:441-458 + gaussian_2d.wgsl:134-156
            const float pcx = mx + sp.extra[4], pcy = my * sp.extra[6] + sp.extra[5];
            const float* T0 = &sp.extra[7]; const float* T1 = &sp.extra[10]; const float* T2 = &sp.extra[13];
            const float hu[3] = {pcx * T2[0] - T0[0], pcx * T2[1] - T0[1], pcx * T2[2] - T0[2]};
            const float hv[3] = {pcy * T2[0] - T1[0], pcy * T2[1] - T1[1], pcy * T2[2] - T1[2]};
            const float px = hu[1] * hv[2] - hu[2] * hv[1];
            const float py = hu[2] * hv[0] - hu[0] * hv[2];
            const float pz = hu[0] * hv[1] - hu[1] * hv[0];
            const float us = px / pz, vs = py / pz;
            const float s3 = us * us + vs * vs;
            const float ex = sp.extra[4] - pcx, ey = sp.extra[5] - pcy;
            const float s2 = 2.0f * (ex * ex + ey * ey);
            power = -(0.5f * std::fmin(s3, s2));
        }
        d.power = power;
        if (power > 0.0f) return d;                      // gaussian.wgsl:468-470
    }
    d.power = power;
    d.covered = true;
    return d;
}

inline float alpha_of(const orc_splat& sp, float power) { return std::fmin(std::exp(power) * sp.op, 0.999f); }

// returns coverage; *alpha = min(exp(power) * opacity, 0.999) where covered
inline bool eval_alpha(const orc_splat& sp, const orc_settings& s, float fx, float fy, float* alpha) {
    const Decision d = decide(sp, s, fx, fy);
    if (!d.covered) return false;
    *alpha = alpha_of(sp, d.power);
    return true;
}

struct Frame {
    std::vector<uint32_t> keys, order;   // order = sorted index (far -> near, culled last)
    std::vector<orc_splat> splats;       // front-to-back rank r -> record
    std::vector<uint32_t> rank_to_id;
    uint32_t n_vis = 0;
};

void build_frame(const Ctx& C, uint32_t n, const float* pos, const float* sh, const float* rot,
                 const float* so, Frame& F) {
    F.keys.resize(n); F.order.resize(n);
    const uint32_t shift = C.plan.shift;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) F.keys[i] = key_of(pos + 4 * i, *C.v, *C.u, shift).key;
    std::iota(F.order.begin(), F.order.end(), 0u);
    const uint32_t* kp = F.keys.data();
    std::stable_sort(F.order.begin(), F.order.end(), [kp](uint32_t a, uint32_t b) { return kp[a] < kp[b]; });
    // visible = in frustum.  At 32-bit keys that is key != 0xFFFFFFFF (gaussian.wgsl:198); at
    // 16/24 bits the vertex stage re-tests the frustum (gaussian.wgsl:212-214): same set.
    uint32_t nv = 0;
    const uint32_t culled = 0xFFFFFFFFu >> shift;
    while (nv < n && F.keys[F.order[nv]] != culled) ++nv;
    F.n_vis = nv;
    F.splats.resize(nv); F.rank_to_id.resize(nv);
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)nv; ++r) {
        const uint32_t id = F.order[nv - 1 - r];
        F.rank_to_id[r] = id;
        project_one(C, pos + 4 * (size_t)id, sh + 48 * (size_t)id, rot + 4 * (size_t)id, so + 4 * (size_t)id, F.splats[r]);
    }
    if (C.s->rasterize_mode == 1u && n >= 2) {
        // gaussian.wgsl:329-349: min from sorted[N-1], max from sorted[1] (literal quirk)
        auto dist = [&](uint32_t id) {
            float pw[4]; const float* p = pos + 4 * (size_t)id;
            mat4_point(C.u->transform, p[0], p[1], p[2], pw);
            const float d[3] = {pw[0] - C.v->world_position[0], pw[1] - C.v->world_position[1], pw[2] - C.v->world_position[2]};
            return std::sqrt(dot3(d, d));
        };
        const float dmin = dist(F.order[n - 1]), dmax = dist(F.order[1]);
        for (uint32_t r = 0; r < nv; ++r) {
            if (F.splats[r].xlo > F.splats[r].xhi) continue;
            float rgb[3];
            depth_to_rgb(dist(F.rank_to_id[r]), dmin, dmax, rgb);
            if (!(C.s->draw_mode == 2u && pos[4 * (size_t)F.rank_to_id[r] + 3] > 0.5f)) {
                F.splats[r].r = rgb[0]; F.splats[r].g = rgb[1]; F.splats[r].b = rgb[2];
            }
        }
    }
}

// a7: per-tile slice of the global order: every splat whose pixel bbox touches the tile, in front-to-back rank
// order.  count[t] .. count[t + 1] is tile t's slice of `entries` (ranks).
void bin_tiles(const Frame& F, int TX, int TY, std::vector<uint64_t>& count, std::vector<uint32_t>& entries) {
    const int NT = TX * TY;
    count.assign((size_t)NT + 1, 0);
    for (uint32_t r = 0; r < F.n_vis; ++r) {
        const orc_splat& sp = F.splats[r];
        if (sp.xlo > sp.xhi) continue;
        for (int ty = sp.ylo / TILE; ty <= sp.yhi / TILE; ++ty)
            for (int tx = sp.xlo / TILE; tx <= sp.xhi / TILE; ++tx) count[(size_t)ty * TX + tx + 1]++;
    }
    for (int t = 0; t < NT; ++t) count[t + 1] += count[t];
    entries.resize(count[NT]);
    std::vector<uint64_t> cur(count.begin(), count.end() - 1);
    for (uint32_t r = 0; r < F.n_vis; ++r) {
        const orc_splat& sp = F.splats[r];
        if (sp.xlo > sp.xhi) continue;
        for (int ty = sp.ylo / TILE; ty <= sp.yhi / TILE; ++ty)
            for (int tx = sp.xlo / TILE; tx <= sp.xhi / TILE; ++tx) entries[cur[(size_t)ty * TX + tx]++] = r;
    }
}

bool make_ctx(Ctx& C, const orc_view* v, const orc_uniform* u, const orc_settings* s) {
    if (!v || !u || !s) return false;
    if (s->radix_sort_depth_bits != 16 && s->radix_sort_depth_bits != 24 && s->radix_sort_depth_bits != 32) return false;
    C.v = v; C.u = u; C.s = s;
    C.W = v->viewport[2]; C.H = v->viewport[3];
    C.Wi = (int)C.W; C.Hi = (int)C.H;
    if (C.Wi <= 0 || C.Hi <= 0) return false;
    C.plan = pass_plan(s->radix_sort_depth_bits);
    return true;
}

}  // namespace

extern "C" {

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

float orc_ln(float x) { return det_ln(x); }

void orc_pass_plan(uint32_t depth_bits, uint32_t* places, uint32_t* shift, uint32_t* parity) {
    const PassPlan p = pass_plan(depth_bits);
    *places = p.places; *shift = p.shift; *parity = p.parity;
}

int orc_keygen(uint32_t n, const float* pos_vis, const orc_view* view, const orc_uniform* u,
               uint32_t depth_bits, uint32_t* keys_out) {
    if (depth_bits != 16 && depth_bits != 24 && depth_bits != 32) return 2;
    const uint32_t shift = pass_plan(depth_bits).shift;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) keys_out[i] = key_of(pos_vis + 4 * i, *view, *u, shift).key;
    return 0;
}

// The literal pass structure of run_radix_sort (src/sort/radix.rs:672-754): per digit place
// (least significant first) count -> exclusive scan -> stable scatter between two ping-pong
// buffers; the parity rule makes the last pass land in the "sorted entries" buffer (index 1).
int orc_radix_sort(uint32_t n, const uint32_t* keys, uint32_t depth_bits, uint32_t* sorted_keys,
                   uint32_t* sorted_index) {
    if (depth_bits != 16 && depth_bits != 24 && depth_bits != 32) return 2;
    const PassPlan plan = pass_plan(depth_bits);
    // buffer 0 = sorted_entry_buffer (what the draw reads), buffer 1 = entry_buffer_b.
    // bind-group parity 0: input 0 -> output 1; parity 1: input 1 -> output 0 (radix.rs:549-562).
    std::vector<uint32_t> kbuf[2], vbuf[2];
    for (int b = 0; b < 2; ++b) { kbuf[b].resize(n); vbuf[b].resize(n); }
    // radix_sort_a fills input_entries of the initial-parity bind group (radix.rs:690-702)
    int src = (plan.parity == 0u) ? 0 : 1;
    for (uint32_t i = 0; i < n; ++i) { kbuf[src][i] = keys[i]; vbuf[src][i] = i; }
    for (uint32_t pass = 0; pass < plan.places; ++pass) {
        const uint32_t par = (pass + plan.parity) % 2u;          // radix.rs:728-731
        if (src != (par == 0u ? 0 : 1)) return 3;                // input of this pass = last output
        const int dst = src ^ 1;
        uint32_t hist[256] = {0};
        for (uint32_t i = 0; i < n; ++i) hist[(kbuf[src][i] >> (8u * pass)) & 255u]++;
        uint32_t sum = 0;
        for (int d = 0; d < 256; ++d) { const uint32_t c = hist[d]; hist[d] = sum; sum += c; }
        for (uint32_t i = 0; i < n; ++i) {
            const uint32_t d = (kbuf[src][i] >> (8u * pass)) & 255u;
            const uint32_t at = hist[d]++;
            kbuf[dst][at] = kbuf[src][i]; vbuf[dst][at] = vbuf[src][i];
        }
        src = dst;
    }
    if (src != 0) return 3;   // tests/radix.rs:65-79: the final pass lands in sorted_entry_buffer
    std::memcpy(sorted_keys, kbuf[0].data(), (size_t)n * 4);
    std::memcpy(sorted_index, vbuf[0].data(), (size_t)n * 4);
    return 0;
}

int orc_stable_sort(uint32_t n, const uint32_t* keys, uint32_t* sorted_index) {
    std::iota(sorted_index, sorted_index + n, 0u);
    std::stable_sort(sorted_index, sorted_index + n, [keys](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
    return 0;
}

void orc_pack_f16(uint32_t n, const float* sh, const float* rot, const float* so,
                  uint32_t* sh_packed, uint32_t* rso_packed) {
    auto pack = [](float upper, float lower) {   // f16.rs:244-252
        return ((uint32_t)f32_to_f16(upper) << 16) | (uint32_t)f32_to_f16(lower);
    };
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) {
        // spherical_harmonics.rs:140-148: even coefficient in the low half
        for (int k = 0; k < 24; ++k) sh_packed[24 * i + k] = pack(sh[48 * i + 2 * k + 1], sh[48 * i + 2 * k]);
        rso_packed[4 * i + 0] = pack(rot[4 * i + 0], rot[4 * i + 1]);   // f16.rs:38-56
        rso_packed[4 * i + 1] = pack(rot[4 * i + 2], rot[4 * i + 3]);
        rso_packed[4 * i + 2] = pack(so[4 * i + 0], so[4 * i + 1]);
        rso_packed[4 * i + 3] = pack(so[4 * i + 2], so[4 * i + 3]);
    }
}

void orc_decode_f16(uint32_t n, const uint32_t* sh_packed, const uint32_t* rso, float* sh, float* rot,
                    float* so) {
    auto hi = [](uint32_t w) { return f16_to_f32((uint16_t)(w >> 16)); };
    auto lo = [](uint32_t w) { return f16_to_f32((uint16_t)(w & 0xFFFFu)); };
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) {
        for (int k = 0; k < 24; ++k) {          // planar.wgsl:117-130
            sh[48 * i + 2 * k] = lo(sh_packed[24 * i + k]);
            sh[48 * i + 2 * k + 1] = hi(sh_packed[24 * i + k]);
        }
        rot[4 * i + 0] = hi(rso[4 * i + 0]); rot[4 * i + 1] = lo(rso[4 * i + 0]);   // planar.wgsl:154-176
        rot[4 * i + 2] = hi(rso[4 * i + 1]); rot[4 * i + 3] = lo(rso[4 * i + 1]);
        so[4 * i + 0] = hi(rso[4 * i + 2]); so[4 * i + 1] = lo(rso[4 * i + 2]);
        so[4 * i + 2] = hi(rso[4 * i + 3]); so[4 * i + 3] = lo(rso[4 * i + 3]);
    }
}

// src/gaussian/covariance.rs:4-41 (compute_covariance_3d, the source of Covariance3dOpacity, f32.rs:238-251): Sigma = M^T M,
// M = S R, R's columns as written there, upper triangle (xx, xy, xz, yy, yz, zz).  glam's Mat3 products accumulate
// column by column: ((a0 b0 + a1 b1) + a2 b2).
void orc_covariance_3d(uint32_t n, const float* rot, const float* so, float* cov6) {
    for (uint32_t g = 0; g < n; ++g) {
        const float* q = rot + 4 * (size_t)g; const float* s3 = so + 4 * (size_t)g;
        float Rm[3][3];
        rotation_rows(q, Rm);                       // Rm[i][j]: row i, column j of R (columns = the written triplets)
        float M[3][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) M[i][j] = s3[i] * Rm[i][j];
        float Sg[3][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
            Sg[i][j] = (M[0][i] * M[0][j] + M[1][i] * M[1][j]) + M[2][i] * M[2][j];
        float* o = cov6 + 6 * (size_t)g;
        o[0] = Sg[0][0]; o[1] = Sg[0][1]; o[2] = Sg[0][2]; o[3] = Sg[1][1]; o[4] = Sg[1][2]; o[5] = Sg[2][2];
    }
}

int orc_project(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                const orc_view* view, const orc_uniform* u, const orc_settings* s, uint32_t count,
                const uint32_t* ids, orc_splat* out) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < (int64_t)count; ++j) {
        const uint32_t id = ids[j];
        if (id >= n) { std::memset(&out[j], 0, sizeof(orc_splat)); set_bbox_empty(out[j]); continue; }
        project_one(C, pos_vis + 4 * (size_t)id, sh + 48 * (size_t)id, rot + 4 * (size_t)id, so + 4 * (size_t)id, out[j]);
    }
    return 0;
}

int orc_render_ref(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                   const orc_view* view, const orc_uniform* u, const orc_settings* s, float* out, int threads) {
    return orc_render_ref_over(n, pos_vis, sh, rot, so, view, u, s, nullptr, out, threads);
}

// The same back-to-front pass over an arbitrary initial target (premultiplied linear RGBA): what the reference's
// Transparent3d item does to the view target it is drawn into (render/mod.rs:398-452, :944-948).  dst_init == NULL is
// the opaque black clear of examples/headless.rs:70; all-zero dst_init yields the layer alone, (C, 1 - T).
int orc_render_ref_over(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                        const orc_view* view, const orc_uniform* u, const orc_settings* s, const float* dst_init,
                        float* out, int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_frame(C, n, pos_vis, sh, rot, so, F);
    const int W = C.Wi, H = C.Hi;
    // clear = opaque black (examples/headless.rs:70); blend = premultiplied "over"
    // (render/mod.rs:944-948) applied far -> near.  Row bands are independent.
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

int orc_render_tiles(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                     const orc_view* view, const orc_uniform* u, const orc_settings* s, float* out,
                     uint32_t* tile_ranges, uint32_t* tile_entries, uint64_t cap, uint64_t* n_pairs,
                     uint32_t* n_vis, uint32_t* rank_to_id, int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_frame(C, n, pos_vis, sh, rot, so, F);
    const int W = C.Wi, H = C.Hi;
    const int TX = (W + TILE - 1) / TILE, TY = (H + TILE - 1) / TILE;
    const int NT = TX * TY;
    std::vector<uint64_t> count;
    std::vector<uint32_t> entries;
    bin_tiles(F, TX, TY, count, entries);
    const uint64_t total = count[NT];
    if (n_pairs) *n_pairs = total;
    if (n_vis) *n_vis = F.n_vis;
    if (rank_to_id) std::memcpy(rank_to_id, F.rank_to_id.data(), (size_t)F.n_vis * 4);
    if (tile_ranges) for (int t = 0; t < NT; ++t) {
        // empty tiles report (0, 0), matching the CUDA range build
        const bool empty = count[t] == count[t + 1];
        tile_ranges[2 * t] = empty ? 0u : (uint32_t)count[t];
        tile_ranges[2 * t + 1] = empty ? 0u : (uint32_t)count[t + 1];
    }
    if (tile_entries) std::memcpy(tile_entries, entries.data(), (size_t)std::min<uint64_t>(total, cap) * 4);
    if (!out) return 0;
#pragma omp parallel for schedule(dynamic, 4)
    for (int t = 0; t < NT; ++t) {
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
            px[0] = cr; px[1] = cg; px[2] = cb; px[3] = 1.0f;   // over opaque black: alpha stays 1
        }
    }
    return 0;
}

int orc_coverage_probe(uint32_t count, const orc_splat* splats, const orc_settings* s, const float* pixel_xy,
                       orc_probe* out) {
    if (!s) return 2;
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < (int64_t)count; ++j) {
        const orc_splat& sp = splats[j];
        const float fx = pixel_xy[2 * j], fy = pixel_xy[2 * j + 1];
        const Decision d = decide(sp, *s, fx, fy), du = decide(sp, *s, fx, fy, false);
        orc_probe& o = out[j];
        o.u = d.u; o.v = d.v; o.mx = d.mx; o.my = d.my; o.Rq = d.Rq; o.power = d.power;
        o.covered = d.covered ? 1u : 0u;
        o.covered_if_unfused = du.covered ? 1u : 0u;
        o.alpha = d.covered ? alpha_of(sp, d.power) : 0.0f;
    }
    return 0;
}

int orc_blend_trace(uint32_t n, const float* pos_vis, const float* sh, const float* rot, const float* so,
                    const orc_view* view, const orc_uniform* u, const orc_settings* s, orc_trace* out, int threads) {
    Ctx C;
    if (!make_ctx(C, view, u, s)) return 2;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    Frame F;
    build_frame(C, n, pos_vis, sh, rot, so, F);
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
                if (!d.covered) continue;
                // f32: exactly render_tiles' step
                const float x32 = std::exp(d.power) * sp.op, a = std::fmin(x32, 0.999f);
                // f64: the same decision and the same stop index, exp of the f32 power in double
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

double orc_cpu_sort_model(uint32_t n, const float* pos_vis, const float* cam, int threads, uint32_t* sorted_index) {
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    struct E { uint32_t key, index; };
    std::vector<E> e(n);
    const auto t0 = std::chrono::steady_clock::now();
    // src/sort/rayon.rs:86-104: key = bits(distance_squared), sort_unstable_by descending
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) {
        const float dx = pos_vis[4 * i] - cam[0], dy = pos_vis[4 * i + 1] - cam[1], dz = pos_vis[4 * i + 2] - cam[2];
        e[i].key = f2u((dx * dx + dy * dy) + dz * dz);
        e[i].index = (uint32_t)i;
    }
#ifdef _OPENMP
    __gnu_parallel::sort(e.begin(), e.end(), [](const E& a, const E& b) { return a.key > b.key; });
#else
    std::sort(e.begin(), e.end(), [](const E& a, const E& b) { return a.key > b.key; });
#endif
    const auto t1 = std::chrono::steady_clock::now();
    if (sorted_index) for (uint32_t i = 0; i < n; ++i) sorted_index[i] = e[i].index;
    return std::chrono::duration<double>(t1 - t0).count();
}

}  // extern "C"
