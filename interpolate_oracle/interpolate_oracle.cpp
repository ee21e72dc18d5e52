// interpolate_oracle.cpp -- see interpolate_oracle.h.  A plain scalar restatement of src/morph/interpolate.wgsl:51-119
// over planar.wgsl's decode (:116-176) and encode (:264-331) of each layout; the compile flags (-ffp-contract=off, no
// fast-math) keep every operation an IEEE f32 round-to-nearest-even one.
#include "interpolate_oracle.h"

#include <cmath>
#include <cstring>

namespace {

uint32_t bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
float from_bits(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

// One gaussian, decoded to f32 (the WGSL getters' view of it)
struct Gaussian {
    float pos[4];      // x, y, z, visibility
    float sh[48];
    float rot[4];      // w, x, y, z (storage order)
    float scale[3];
    float opacity;
    float cov[6];
};

float mix(float a, float b, float t) {
    const float omt = 1.0f - t;
    const float l = a * omt;
    const float r = b * t;
    return l + r;
}

// interpolate.wgsl:59-65
void normalize_quaternion(float q[4]) {
    float l2 = q[0] * q[0];
    l2 = l2 + q[1] * q[1];
    l2 = l2 + q[2] * q[2];
    l2 = l2 + q[3] * q[3];
    if (l2 <= 0.0f) {
        q[0] = 0.0f; q[1] = 0.0f; q[2] = 0.0f; q[3] = 1.0f;
        return;
    }
    const float s = std::sqrt(l2);
    for (int k = 0; k < 4; ++k) q[k] = q[k] / s;
}

float lo(uint32_t w) { return orc_half_to_float((uint16_t)(w & 0xFFFFu)); }
float hi(uint32_t w) { return orc_half_to_float((uint16_t)(w >> 16)); }
// pack2x16float(vec2(low, high))
uint32_t pack2x16(float low, float high) { return ((uint32_t)orc_float_to_half(high) << 16) | orc_float_to_half(low); }

Gaussian decode(int layout, const void* const p[4], uint32_t i) {
    Gaussian g = {};
    std::memcpy(g.pos, static_cast<const float*>(p[0]) + (size_t)i * 4, 16);
    if (layout == ORC_INTERP_F32) {
        std::memcpy(g.sh, static_cast<const float*>(p[1]) + (size_t)i * 48, 192);
        std::memcpy(g.rot, static_cast<const float*>(p[2]) + (size_t)i * 4, 16);
        const float* so = static_cast<const float*>(p[3]) + (size_t)i * 4;
        g.scale[0] = so[0]; g.scale[1] = so[1]; g.scale[2] = so[2]; g.opacity = so[3];
        return g;
    }
    const uint32_t* sh = static_cast<const uint32_t*>(p[1]) + (size_t)i * 24;
    for (int k = 0; k < 24; ++k) { g.sh[2 * k] = lo(sh[k]); g.sh[2 * k + 1] = hi(sh[k]); }   // planar.wgsl:117-130
    const uint32_t* w = static_cast<const uint32_t*>(p[2]) + (size_t)i * 4;
    if (layout == ORC_INTERP_F16_COV) {   // planar.wgsl:133-152
        for (int k = 0; k < 3; ++k) { g.cov[2 * k] = hi(w[k]); g.cov[2 * k + 1] = lo(w[k]); }
        g.opacity = hi(w[3]);
    } else {                              // planar.wgsl:154-176
        g.rot[0] = hi(w[0]); g.rot[1] = lo(w[0]); g.rot[2] = hi(w[1]); g.rot[3] = lo(w[1]);
        g.scale[0] = hi(w[2]); g.scale[1] = lo(w[2]); g.scale[2] = hi(w[3]);
        g.opacity = lo(w[3]);
    }
    return g;
}

void encode(int layout, const Gaussian& g, void* const p[4], uint32_t i) {
    std::memcpy(static_cast<float*>(p[0]) + (size_t)i * 4, g.pos, 16);
    if (layout == ORC_INTERP_F32) {
        std::memcpy(static_cast<float*>(p[1]) + (size_t)i * 48, g.sh, 192);
        std::memcpy(static_cast<float*>(p[2]) + (size_t)i * 4, g.rot, 16);
        float* so = static_cast<float*>(p[3]) + (size_t)i * 4;
        so[0] = g.scale[0]; so[1] = g.scale[1]; so[2] = g.scale[2]; so[3] = g.opacity;
        return;
    }
    uint32_t* sh = static_cast<uint32_t*>(p[1]) + (size_t)i * 24;
    for (int k = 0; k < 24; ++k) sh[k] = pack2x16(g.sh[2 * k], g.sh[2 * k + 1]);            // planar.wgsl:272-283
    uint32_t* w = static_cast<uint32_t*>(p[2]) + (size_t)i * 4;
    if (layout == ORC_INTERP_F16_COV) {   // planar.wgsl:286-296
        for (int k = 0; k < 3; ++k) w[k] = pack2x16(g.cov[2 * k + 1], g.cov[2 * k]);
        w[3] = pack2x16(0.0f, g.opacity);
    } else {                              // planar.wgsl:306-317
        w[0] = pack2x16(g.rot[1], g.rot[0]);
        w[1] = pack2x16(g.rot[3], g.rot[2]);
        w[2] = pack2x16(g.scale[1], g.scale[0]);
        w[3] = pack2x16(g.opacity, g.scale[2]);
    }
}

}  // namespace

extern "C" {

float orc_half_to_float(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    if (e == 0x1F) return from_bits(sign | 0x7F800000u | (m << 13));          // inf, NaN (payload kept)
    if (e != 0) return from_bits(sign | ((e + 112u) << 23) | (m << 13));     // normal: exponent - 15 + 127
    // zero or subnormal: m * 2^-24, exact in f32
    const float v = (float)m * from_bits(0x33800000u);                        // 2^-24
    return sign ? -v : v;
}

uint16_t orc_float_to_half(float f) {
    const uint32_t x = bits(f), a = x & 0x7FFFFFFFu;
    const uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
    if (a > 0x7F800000u) return sign | 0x7E00u | (uint16_t)((a >> 13) & 0x3FFu);   // NaN (quiet)
    if (a >= 0x477FF000u) return sign | 0x7C00u;     // >= 65520 (the tie above 65504 rounds to even: up) and inf
    if (a >= 0x38800000u) {                          // normal half (>= 2^-14)
        uint32_t h = ((((a >> 23) - 112u) << 10) | ((a & 0x7FFFFFu) >> 13));
        const uint32_t rem = a & 0x1FFFu;
        if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;   // (a carry moves into the exponent, as it should)
        return sign | (uint16_t)h;
    }
    if (a <= 0x33000000u) return sign;               // <= 2^-25: rounds to zero (2^-25 itself is a tie to even 0)
    // subnormal half: units of 2^-24
    const uint32_t e = a >> 23, m = (a & 0x7FFFFFu) | 0x800000u, shift = 126u - e;
    uint32_t h = m >> shift;
    const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1u);
    if (rem > half || (rem == half && (h & 1u))) ++h;
    return sign | (uint16_t)h;
}

int orc_interp_factor(float time, float time_start, float time_stop, float* t) {
    if (!std::isfinite(time) || !std::isfinite(time_start) || !std::isfinite(time_stop)) return -1;
    // interpolate.wgsl:51-57
    const float duration = time_stop - time_start;
    float f;
    if (std::fabs(duration) < 1e-6f) {
        f = time >= time_stop ? 1.0f : 0.0f;
    } else {
        f = (time - time_start) / duration;
        if (f < 0.0f) f = 0.0f;     // clamp(f, 0, 1) = min(max(f, 0), 1); -0 is not < 0 and stays -0
        if (f > 1.0f) f = 1.0f;
    }
    if (std::isnan(f)) return -1;
    *t = f;
    return 0;
}

void orc_interp(uint32_t n, int layout, float t, const void* const lhs[4], const void* const rhs[4], void* const out[4]) {
    for (uint32_t i = 0; i < n; ++i) {
        const Gaussian l = decode(layout, lhs, i), r = decode(layout, rhs, i);
        Gaussian o = {};
        for (int k = 0; k < 4; ++k) o.pos[k] = mix(l.pos[k], r.pos[k], t);        // :82-89
        for (int k = 0; k < 48; ++k) o.sh[k] = mix(l.sh[k], r.sh[k], t);          // :91-96
        if (layout == ORC_INTERP_F16_COV) {                                        // :98-105
            for (int k = 0; k < 6; ++k) o.cov[k] = mix(l.cov[k], r.cov[k], t);
        } else {                                                                   // :107-117
            for (int k = 0; k < 4; ++k) o.rot[k] = mix(l.rot[k], r.rot[k], t);
            normalize_quaternion(o.rot);
            for (int k = 0; k < 3; ++k) o.scale[k] = mix(l.scale[k], r.scale[k], t);
        }
        o.opacity = mix(l.opacity, r.opacity, t);
        encode(layout, o, out, i);
    }
}

}  // extern "C"
