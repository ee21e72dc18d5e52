// project_math.cuh -- the bit-exact part of the per-gaussian maths (key-gen + projection).
//
// Translation units including this header are compiled with -fmad=false: every a*b+c is a
// rounded multiply followed by a rounded add, in the order written, exactly as the CPU oracle
// evaluates it (-ffp-contract=off).  Division and sqrt are IEEE (nvcc defaults
// -prec-div=true -prec-sqrt=true); no fast-math.  This is what makes sort keys, projected
// records, pixel bounding boxes and therefore tile ranges bit-identical to the oracle.
#pragma once
#include "common.cuh"

namespace bgs {

// M * (x,y,z,1), summed ((m0*x + m1*y) + m2*z) + m3.  Reference: WGSL mat4x4 * vec4
// (radix.wgsl:88, transform.wgsl:6, helpers.wgsl:18).
__device__ __forceinline__ void mat4_point(const float* m, float x, float y, float z, float out[4]) {
#pragma unroll
    for (int r = 0; r < 4; ++r) out[r] = ((m[0 + r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r];
}
__device__ __forceinline__ void mat4_dir(const float* m, float x, float y, float z, float out[4]) {
#pragma unroll
    for (int r = 0; r < 4; ++r) out[r] = (m[0 + r] * x + m[4 + r] * y) + m[8 + r] * z;
}

// Key-gen's world position (radix.wgsl:89-90): M * (p, 1), skipping the multiply under an identity model matrix (the
// common case) when p is finite, where x*1 + y*0 + z*0 + 0 == x bit for bit -- except that a -0 coordinate comes out
// +0.  The sign of that zero changes no key and no visibility decision, but it does reach the projection's records,
// so the projection keeps the full multiply.
__device__ __forceinline__ void keygen_world_pos(const FrameConsts& c, float4 p, float pw[4]) {
    if (c.model_identity && (fabsf(p.x) + fabsf(p.y)) + fabsf(p.z) < __uint_as_float(0x7F800000u)) {
        pw[0] = p.x; pw[1] = p.y; pw[2] = p.z; pw[3] = 1.0f;
    } else {
        mat4_point(c.model, p.x, p.y, p.z, pw);
    }
}

// transform.wgsl:5-8, literal: world_to_clip, clip_from_world (p, 1) with every lane divided (IEEE) by w + 1e-9.
// (Callers that read only some lanes leave the other divisions to dead-code elimination.)
__device__ __forceinline__ void world_to_clip(const FrameConsts& c, const float pw[3], float out[4]) {
    float cl[4];
    mat4_point(c.clip_from_world, pw[0], pw[1], pw[2], cl);
    const float den = cl[3] + 0.000000001f;
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = cl[i] / den;
}

// transform.wgsl:10-14, literal: in_frustum of world_to_clip's x, y, z.
__device__ __forceinline__ bool in_frustum(const FrameConsts& c, const float pw[3], float ndc[2]) {
    float h[4];
    world_to_clip(c, pw, h);
    const float nx = h[0], ny = h[1], nz = h[2];
    ndc[0] = nx; ndc[1] = ny;
    return fabsf(nx) < 1.1f && fabsf(ny) < 1.1f && fabsf(nz - 0.5f) < 0.5f;
}

// bgs_render_depth_test's splat depth (include/bgs.h): world_to_clip's z over its w.
__device__ __forceinline__ float splat_depth(const FrameConsts& c, const float pw[3]) {
    float h[4];
    world_to_clip(c, pw, h);
    return h[2] / h[3];
}

// in_frustum's decision, cheaper, for key-gen (which needs no ndc): one approximate reciprocal (|error| < 4e-7
// relative) decides every gaussian whose ndc is not within 1e-4 of a frustum bound; the few that are fall back to
// the exact divisions.  Denominators outside [1e-30, 1e30] (rcp.approx flushes) also fall back.
__device__ __forceinline__ bool in_frustum_fast(const FrameConsts& c, const float pw[3]) {
    float cl[4];
    mat4_point(c.clip_from_world, pw[0], pw[1], pw[2], cl);
    const float den = cl[3] + 0.000000001f;
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(den));
    const float ax = fabsf(cl[0] * rc), ay = fabsf(cl[1] * rc), z = cl[2] * rc;
    const float ad = fabsf(den);
    const bool sure_in = ax < 1.0999f && ay < 1.0999f && z > 1e-6f && z < 0.9999f;
    const bool sure_out = ax > 1.1001f || ay > 1.1001f || z < -1e-6f || z > 1.0001f;
    const bool den_ok = ad > 1e-30f && ad < 1e30f;
    if (den_ok && (sure_in || sure_out)) return sure_in;
    float ndc[2];
    return in_frustum(c, pw, ndc);
}

// |pw - cam|^2 (radix.wgsl:92-93): what the depth key encodes; its square root is the Depth colour source's depth.
__device__ __forceinline__ float cam_dist2(const FrameConsts& c, const float pw[3]) {
    const float dx = pw[0] - c.cam[0], dy = pw[1] - c.cam[1], dz = pw[2] - c.cam[2];
    return (dx * dx + dy * dy) + dz * dz;
}

// radix.wgsl:94-99: the depth key, far first; a culled gaussian's is all ones.
__device__ __forceinline__ uint32_t depth_key(const FrameConsts& c, bool visible, float d2) {
    uint32_t key = 0xFFFFFFFFu;
    if (visible) key = 0xFFFFFFFFu - __float_as_uint(d2);
    return key >> c.key_shift;
}

// Fixed-series natural log in f64 (the policy replacement for WGSL log(), gaussian.wgsl:229):
// x = m 2^e, m in [sqrt(1/2), sqrt 2); s = (m-1)/(m+1); ln x = e ln2 + 2 s P(s^2), rounded to f32.
__device__ __forceinline__ float det_ln(float xf) {
    if (xf != xf) return xf;
    if (xf < 0.0f) return __uint_as_float(0x7FC00000u);
    if (xf == 0.0f) return __uint_as_float(0xFF800000u);
    if (xf == __uint_as_float(0x7F800000u)) return xf;
    const double x = (double)xf;
    unsigned long long bits = (unsigned long long)__double_as_longlong(x);
    int e = (int)((bits >> 52) & 0x7FFull) - 1023;
    bits = (bits & 0x000FFFFFFFFFFFFFull) | 0x3FF0000000000000ull;
    double m = __longlong_as_double((long long)bits);
    if (m > 1.4142135623730951) { m = __dmul_rn(m, 0.5); e += 1; }
    const double s = __ddiv_rn(__dsub_rn(m, 1.0), __dadd_rn(m, 1.0));
    const double z = __dmul_rn(s, s);
    double p = 1.0 / 23.0;
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 21.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 19.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 17.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 15.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 13.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 11.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 9.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 7.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 5.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0 / 3.0);
    p = __dadd_rn(__dmul_rn(p, z), 1.0);
    const double r = __dadd_rn(__dmul_rn((double)e, 0.6931471805599453), __dmul_rn(2.0, __dmul_rn(s, p)));
    return (float)r;   // cvt.rn.f32.f64
}

// Fixed-series exp in f64 (the policy replacement for WGSL exp, gaussian_4d.wgsl's marginal_t), shared with the oracle:
// x = k ln2 + r, k = rint(x / ln2), r = x - k ln2 (|r| <= 0.35); e^r by its Taylor polynomial to degree 16 (remainder
// < 1e-20), coefficients 1 / j! built by repeated division; times 2^k exactly; rounded to f32.  Below -110 the f32
// result is 0, above 89 it is +inf.
__device__ __forceinline__ float det_exp(float xf) {
    if (xf != xf) return xf;
    if (xf < -110.0f) return 0.0f;
    if (xf > 89.0f) return __uint_as_float(0x7F800000u);
    const double x = (double)xf;
    const double k = rint(__dmul_rn(x, 1.4426950408889634));
    const double r = __dsub_rn(x, __dmul_rn(k, 0.6931471805599453));
    double c[17];
    c[0] = 1.0;
#pragma unroll
    for (int j = 1; j <= 16; ++j) c[j] = c[j - 1] / (double)j;   // (folded by the compiler, IEEE)
    double p = c[16];
#pragma unroll
    for (int j = 15; j >= 0; --j) p = __dadd_rn(__dmul_rn(p, r), c[j]);
    const double scale = __longlong_as_double((long long)((unsigned long long)((int)k + 1023) << 52));
    return (float)__dmul_rn(p, scale);   // cvt.rn.f32.f64
}

// Fixed-series cos in f64 (the policy replacement for WGSL cos, spherindrical_harmonics.wgsl's time terms), shared with
// the oracle: r = x - k 2pi, k = rint(x / 2pi) (|r| <= pi + rounding); cos r = P(r^2) by its Taylor polynomial to degree
// 36 (remainder < 1e-24), coefficients (-1)^j / (2j)! built by repeated division; rounded to f32.  Not finite: NaN.
__device__ __forceinline__ float det_cos(float xf) {
    if (!(fabsf(xf) < __uint_as_float(0x7F800000u))) return __uint_as_float(0x7FC00000u);
    const double x = (double)xf;
    const double k = rint(__dmul_rn(x, 0.15915494309189535));
    const double r = __dsub_rn(x, __dmul_rn(k, 6.283185307179586));
    const double z = __dmul_rn(r, r);
    double c[19];
    c[0] = 1.0;
#pragma unroll
    for (int j = 1; j <= 18; ++j) c[j] = -c[j - 1] / (double)((2 * j - 1) * (2 * j));   // (folded, IEEE)
    double p = c[18];
#pragma unroll
    for (int j = 17; j >= 0; --j) p = __dadd_rn(__dmul_rn(p, z), c[j]);
    return (float)p;
}

}  // namespace bgs
