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

// transform.wgsl:5-14, literal: world_to_clip (three IEEE divisions by w + 1e-9) and in_frustum.
__device__ __forceinline__ bool in_frustum(const FrameConsts& c, const float pw[3], float ndc[2]) {
    float cl[4];
    mat4_point(c.clip_from_world, pw[0], pw[1], pw[2], cl);
    const float den = cl[3] + 0.000000001f;
    const float nx = cl[0] / den, ny = cl[1] / den, nz = cl[2] / den;
    ndc[0] = nx; ndc[1] = ny;
    return fabsf(nx) < 1.1f && fabsf(ny) < 1.1f && fabsf(nz - 0.5f) < 0.5f;
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

}  // namespace bgs
