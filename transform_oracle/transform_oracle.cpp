// transform_oracle.cpp -- see transform_oracle.h.  A plain scalar restatement of include/bgs.h's bgs_cloud_transform over
// the upload planes of each layout; the compile flags (-ffp-contract=off, no fast-math) keep every f32 operation one
// IEEE round-to-nearest-even operation.
#include "transform_oracle.h"

#include <cmath>
#include <cstring>

namespace {

float half_to_float(uint16_t h) { _Float16 v; std::memcpy(&v, &h, 2); return (float)v; }
uint16_t float_to_half(float f) { const _Float16 v = (_Float16)f; uint16_t h; std::memcpy(&h, &v, 2); return h; }
float lo(uint32_t w) { return half_to_float((uint16_t)(w & 0xFFFFu)); }
float hi(uint32_t w) { return half_to_float((uint16_t)(w >> 16)); }
uint32_t pack(float high, float low) { return ((uint32_t)float_to_half(high) << 16) | float_to_half(low); }

// the renderer's sixteen basis functions (spherical_harmonics.wgsl's polynomials and constants), in f64
void basis16(const double d[3], double b[16]) {
    static const double k[16] = {0.28209479177387814, -0.4886025119029199, 0.4886025119029199, -0.4886025119029199,
                                 1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                                 0.5462742152960396, -0.5900435899266435, 2.890611442640554, -0.4570457994644658,
                                 0.3731763325901154, -0.4570457994644658, 1.445305721320277, -0.5900435899266435};
    const double x = d[0], y = d[1], z = d[2], xx = x * x, yy = y * y, zz = z * z;
    const double p[16] = {1.0, y, z, x, x * y, y * z, 2.0 * zz - xx - yy, x * z, xx - yy, y * (3.0 * xx - yy), x * y * z,
                          y * (4.0 * zz - xx - yy), z * (2.0 * zz - 3.0 * xx - 3.0 * yy), x * (4.0 * zz - xx - yy), z * (xx - yy),
                          x * (xx - 3.0 * yy)};
    for (int i = 0; i < 16; ++i) b[i] = k[i] * p[i];
}

// Shepperd's method, normalised, w >= 0 (bgs.h); q in f64
void shepperd(const double R[3][3], double q[4]) {
    const double tr = (R[0][0] + R[1][1]) + R[2][2];
    const double c[4] = {tr, R[0][0], R[1][1], R[2][2]};
    int b = 0;
    for (int k = 1; k < 4; ++k)
        if (c[k] > c[b]) b = k;
    double t, f;
    switch (b) {
    case 0:
        t = 0.5 * std::sqrt(1.0 + tr); f = 0.25 / t;
        q[0] = t; q[1] = (R[2][1] - R[1][2]) * f; q[2] = (R[0][2] - R[2][0]) * f; q[3] = (R[1][0] - R[0][1]) * f;
        break;
    case 1:
        t = 0.5 * std::sqrt(((1.0 + R[0][0]) - R[1][1]) - R[2][2]); f = 0.25 / t;
        q[1] = t; q[0] = (R[2][1] - R[1][2]) * f; q[2] = (R[0][1] + R[1][0]) * f; q[3] = (R[0][2] + R[2][0]) * f;
        break;
    case 2:
        t = 0.5 * std::sqrt(((1.0 - R[0][0]) + R[1][1]) - R[2][2]); f = 0.25 / t;
        q[2] = t; q[0] = (R[0][2] - R[2][0]) * f; q[1] = (R[0][1] + R[1][0]) * f; q[3] = (R[1][2] + R[2][1]) * f;
        break;
    default:
        t = 0.5 * std::sqrt(((1.0 - R[0][0]) - R[1][1]) + R[2][2]); f = 0.25 / t;
        q[3] = t; q[0] = (R[1][0] - R[0][1]) * f; q[1] = (R[0][2] + R[2][0]) * f; q[2] = (R[1][2] + R[2][1]) * f;
    }
    const double n = std::sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
    const double sg = q[0] < 0.0 ? -1.0 : 1.0;
    for (int k = 0; k < 4; ++k) q[k] = sg * q[k] / n;
}

struct Params {
    float m[16], q[4], s;
    float E[4][49];   // E[l], l = 1..3
};

bool params(const float* M, Params* P) {
    for (int k = 0; k < 16; ++k)
        if (!std::isfinite(M[k])) return false;
    if (!(M[3] == 0.0f && M[7] == 0.0f && M[11] == 0.0f && M[15] == 1.0f)) return false;
    double col[3][3];   // col[j] = column j of the 3x3 block
    for (int j = 0; j < 3; ++j)
        for (int i = 0; i < 3; ++i) col[j][i] = M[4 * j + i];
    double g[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) g[i][j] = (col[i][0] * col[j][0] + col[i][1] * col[j][1]) + col[i][2] * col[j][2];
    const double s2 = ((g[0][0] + g[1][1]) + g[2][2]) / 3.0;
    if (!(s2 > 0.0)) return false;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            if (!(std::fabs(g[i][j] - (i == j ? s2 : 0.0)) <= 1e-5 * s2)) return false;
    // det = c0 . (c1 x c2)
    const double cr[3] = {col[1][1] * col[2][2] - col[1][2] * col[2][1], col[1][2] * col[2][0] - col[1][0] * col[2][2],
                          col[1][0] * col[2][1] - col[1][1] * col[2][0]};
    if (!(col[0][0] * cr[0] + col[0][1] * cr[1] + col[0][2] * cr[2] > 0.0)) return false;
    const double s = std::sqrt(s2);
    double R[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = col[j][i] / s;
    double q[4];
    shepperd(R, q);
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double Rq[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                          2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                          2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
    std::memcpy(P->m, M, 64);
    for (int k = 0; k < 4; ++k) P->q[k] = (float)q[k];
    P->s = (float)s;
    for (int l = 1; l <= 3; ++l) {
        double E[49];
        orc_xf_sh_matrix(Rq, l, E);
        for (int k = 0; k < (2 * l + 1) * (2 * l + 1); ++k) P->E[l][k] = (float)E[k];
    }
    return true;
}

// f32 arithmetic, one rounding per operation
float mul(float a, float b) { return a * b; }
float add(float a, float b) { return a + b; }
float sub(float a, float b) { return a - b; }

void quat(const float a[4], const float b[4], float r[4]) {
    r[0] = sub(sub(sub(mul(a[0], b[0]), mul(a[1], b[1])), mul(a[2], b[2])), mul(a[3], b[3]));
    r[1] = sub(add(add(mul(a[0], b[1]), mul(a[1], b[0])), mul(a[2], b[3])), mul(a[3], b[2]));
    r[2] = add(add(sub(mul(a[0], b[2]), mul(a[1], b[3])), mul(a[2], b[0])), mul(a[3], b[1]));
    r[3] = add(sub(add(mul(a[0], b[3]), mul(a[1], b[2])), mul(a[2], b[1])), mul(a[3], b[0]));
}

// A Sigma A^T, A[i][j] = m[4 j + i]
void cov(const float* m, const float c[6], float o[6]) {
    const float S[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
    float X[3][3], T[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) X[i][j] = add(add(mul(m[i], S[0][j]), mul(m[4 + i], S[1][j])), mul(m[8 + i], S[2][j]));
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T[i][j] = add(add(mul(X[i][0], m[j]), mul(X[i][1], m[4 + j])), mul(X[i][2], m[8 + j]));
    o[0] = T[0][0]; o[1] = T[1][0]; o[2] = T[2][0]; o[3] = T[1][1]; o[4] = T[2][1]; o[5] = T[2][2];
}

uint32_t sh_floats(uint32_t d) { return d == 0 ? 4u : d == 1 ? 12u : d == 2 ? 28u : 48u; }

}  // namespace

extern "C" {

void orc_xf_sh_matrix(const double* R, int l, double* E) {
    // least squares Y E = Z over 100 directions (a Fibonacci sphere of its own), solved through the normal equations by
    // Gaussian elimination with partial pivoting and back substitution
    const int m = 2 * l + 1, k0 = l * l;
    const int N = 100;
    double A[7][7] = {}, B[7][7] = {};
    for (int k = 0; k < N; ++k) {
        const double z = -1.0 + (2.0 * k + 1.0) / N, r = std::sqrt(1.0 - z * z);
        const double phi = k * M_PI * (3.0 - std::sqrt(5.0)) + 0.3;
        const double d[3] = {r * std::cos(phi), r * std::sin(phi), z};
        double rtd[3];
        for (int i = 0; i < 3; ++i) rtd[i] = R[0 * 3 + i] * d[0] + R[1 * 3 + i] * d[1] + R[2 * 3 + i] * d[2];
        double y[16], yr[16];
        basis16(d, y);
        basis16(rtd, yr);
        for (int i = 0; i < m; ++i)
            for (int j = 0; j < m; ++j) {
                A[i][j] += y[k0 + i] * y[k0 + j];
                B[i][j] += y[k0 + i] * yr[k0 + j];
            }
    }
    for (int c = 0; c < m; ++c) {
        int p = c;
        for (int r = c + 1; r < m; ++r)
            if (std::fabs(A[r][c]) > std::fabs(A[p][c])) p = r;
        for (int j = 0; j < m; ++j) { std::swap(A[c][j], A[p][j]); std::swap(B[c][j], B[p][j]); }
        for (int r = c + 1; r < m; ++r) {
            const double f = A[r][c] / A[c][c];
            for (int j = 0; j < m; ++j) { A[r][j] -= f * A[c][j]; B[r][j] -= f * B[c][j]; }
        }
    }
    for (int c = m - 1; c >= 0; --c)
        for (int j = 0; j < m; ++j) {
            double v = B[c][j];
            for (int k = c + 1; k < m; ++k) v -= A[c][k] * E[k * m + j];
            E[c * m + j] = v / A[c][c];
        }
    for (int k = 0; k < m * m; ++k)
        if (std::fabs(E[k]) < 0x1p-40) E[k] = 0.0;
}

int orc_xf_params(const float* M, float* q, float* s, float* E1, float* E2, float* E3) {
    Params P;
    if (!params(M, &P)) return 1;
    if (q) std::memcpy(q, P.q, 16);
    if (s) *s = P.s;
    if (E1) std::memcpy(E1, P.E[1], 9 * 4);
    if (E2) std::memcpy(E2, P.E[2], 25 * 4);
    if (E3) std::memcpy(E3, P.E[3], 49 * 4);
    return 0;
}

int orc_xf_apply(uint32_t n, int layout, uint32_t d, const float* M, uint32_t mode, void* const* planes, double* sh_bound) {
    Params P;
    if (!params(M, &P)) return 1;
    const uint32_t S = sh_floats(d);
    const bool f16 = layout != ORC_XF_F32;
    float* pos = static_cast<float*>(planes[0]);
    for (uint32_t i = 0; i < n; ++i) {
        float* p = pos + (size_t)i * 4;
        double* bound = sh_bound ? sh_bound + (size_t)i * S : nullptr;
        if (bound)
            for (uint32_t h = 0; h < S; ++h) bound[h] = 0.0;
        if (mode == 1 && p[3] < 0.5f) continue;
        const float x = p[0], y = p[1], z = p[2];
        for (int r = 0; r < 3; ++r) p[r] = add(add(add(mul(M[r], x), mul(M[4 + r], y)), mul(M[8 + r], z)), M[12 + r]);
        // the SH lanes as floats, read and written through these two
        float* shf = f16 ? nullptr : static_cast<float*>(planes[1]) + (size_t)i * S;
        uint32_t* shw = f16 ? static_cast<uint32_t*>(planes[1]) + (size_t)i * (S / 2) : nullptr;
        auto get = [&](uint32_t h) { return f16 ? ((h & 1) ? hi(shw[h / 2]) : lo(shw[h / 2])) : shf[h]; };
        auto set = [&](uint32_t h, float v) {
            if (!f16) { shf[h] = v; return; }
            const uint32_t hv = float_to_half(v);
            shw[h / 2] = (h & 1) ? ((shw[h / 2] & 0xFFFFu) | (hv << 16)) : ((shw[h / 2] & 0xFFFF0000u) | hv);
        };
        for (uint32_t l = 1; l <= d; ++l) {
            const uint32_t m = 2 * l + 1, k0 = l * l;
            const float* E = P.E[l];
            for (uint32_t ch = 0; ch < 3; ++ch) {
                float in[7];
                for (uint32_t j = 0; j < m; ++j) in[j] = get(3 * (k0 + j) + ch);
                for (uint32_t a = 0; a < m; ++a) {
                    float acc = mul(E[a * m], in[0]);
                    double b = std::fabs((double)E[a * m] * in[0]);
                    for (uint32_t j = 1; j < m; ++j) {
                        acc = add(acc, mul(E[a * m + j], in[j]));
                        b += std::fabs((double)E[a * m + j] * in[j]);
                    }
                    set(3 * (k0 + a) + ch, acc);
                    if (bound) bound[3 * (k0 + a) + ch] = b;
                }
            }
        }
        if (layout == ORC_XF_F32) {
            float* q = static_cast<float*>(planes[2]) + (size_t)i * 4;
            float* so = static_cast<float*>(planes[3]) + (size_t)i * 4;
            const float b[4] = {q[0], q[1], q[2], q[3]};
            quat(P.q, b, q);
            for (int k = 0; k < 3; ++k) so[k] = mul(P.s, so[k]);
        } else {
            uint32_t* w = static_cast<uint32_t*>(planes[2]) + (size_t)i * 4;
            if (layout == ORC_XF_F16) {
                const float b[4] = {hi(w[0]), lo(w[0]), hi(w[1]), lo(w[1])};
                float r[4];
                quat(P.q, b, r);
                const float sx = mul(P.s, hi(w[2])), sy = mul(P.s, lo(w[2])), sz = mul(P.s, hi(w[3]));
                w[0] = pack(r[0], r[1]);
                w[1] = pack(r[2], r[3]);
                w[2] = pack(sx, sy);
                w[3] = ((uint32_t)float_to_half(sz) << 16) | (w[3] & 0xFFFFu);
            } else {
                const float c[6] = {hi(w[0]), lo(w[0]), hi(w[1]), lo(w[1]), hi(w[2]), lo(w[2])};
                float o[6];
                cov(M, c, o);
                w[0] = pack(o[0], o[1]);
                w[1] = pack(o[2], o[3]);
                w[2] = pack(o[4], o[5]);
            }
        }
    }
    return 0;
}

}  // extern "C"
