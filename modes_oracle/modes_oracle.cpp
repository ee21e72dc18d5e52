// modes_oracle.cpp -- see modes_oracle.h.  Compiled with -ffp-contract=off: every a * b + c below is two roundings.
#include "modes_oracle.h"

#include <cmath>
#include <cstring>

namespace {

const float FRAC_PI_3_F = 1.0471975512f;   // bevy_render::maths, rounded to f32
const float PI_2_F = 6.28318530718f;

void hsv_to_rgb(float h, float s, float v, float rgb[3]) {
    const float hk = h / FRAC_PI_3_F, vs = v * s;
    const float base[3] = {5.0f, 3.0f, 1.0f};
    for (int c = 0; c < 3; ++c) {
        const float x = base[c] + hk;
        const float k = x - 6.0f * std::trunc(x / 6.0f);   // WGSL f32 %, not fmodf
        rgb[c] = v - vs * std::fmax(0.0f, std::fmin(k, std::fmin(4.0f - k, 1.0f)));
    }
}

bool sign_bit(float f) {
    uint32_t b;
    std::memcpy(&b, &f, 4);
    return (b >> 31) != 0;
}

// t = min / max of |y|, |x|; above tan(pi/8) atan t = pi/4 + atan((t - 1) / (t + 1)); atan u = u P(u^2), 22 odd terms
float det_atan2(float yf, float xf) {
    if (std::isnan(yf) || std::isnan(xf)) return std::nanf("");
    const double ay = std::fabs((double)yf), ax = std::fabs((double)xf);
    const bool steep = ay > ax;
    double t;
    if (ax == ay) t = ax == 0.0 ? 0.0 : 1.0;
    else t = steep ? ax / ay : ay / ax;
    double base = 0.0, u = t;
    if (t > 0.41421356237309503) { base = 0.7853981633974483; u = (t - 1.0) / (t + 1.0); }
    const double z = u * u;
    double p = -1.0 / 43.0;
    for (int k = 20; k >= 0; --k) p = p * z + (k & 1 ? -1.0 : 1.0) / (double)(2 * k + 1);
    double r = base + u * p;
    if (steep) r = 1.5707963267948966 - r;
    if (sign_bit(xf)) r = 3.141592653589793 - r;
    if (sign_bit(yf)) r = -r;
    return (float)r;
}

void mat4_point(const float* m, float x, float y, float z, float out[4]) {
    for (int r = 0; r < 4; ++r) out[r] = ((m[0 + r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r];
}

}  // namespace

extern "C" {

void mo_hsv_to_rgb(uint32_t n, const float* h, const float* s, const float* v, float* rgb_out) {
    for (uint32_t i = 0; i < n; ++i) hsv_to_rgb(h[i], s[i], v[i], rgb_out + 3 * (size_t)i);
}

void mo_atan2(uint32_t n, const float* y, const float* x, float* out) {
    for (uint32_t i = 0; i < n; ++i) out[i] = det_atan2(y[i], x[i]);
}

// classification.wgsl:9-27 behind gaussian.wgsl:315-328
void mo_class_colour(uint32_t n, const float* sh_rgb, const float* vis, uint32_t num_classes, float* rgb_out) {
    for (uint32_t i = 0; i < n; ++i) {
        float* o = rgb_out + 3 * (size_t)i;
        const float* sh = sh_rgb + 3 * (size_t)i;
        if (vis[i] < 2.0f) { o[0] = sh[0]; o[1] = sh[1]; o[2] = sh[2]; continue; }
        const float hue = ((vis[i] - 2.0f) / (float)num_classes) * 6.283185307f;
        float h[3];
        hsv_to_rgb(hue, 1.0f, 1.0f, h);
        for (int c = 0; c < 3; ++c) o[c] = sh[c] * (1.0f - 0.5f) + h[c] * 0.5f;
    }
}

// optical_flow.wgsl:16-53 behind gaussian.wgsl:201,369-375
void mo_flow_colour(uint32_t n, const float* pos, const float* model, const float* clip, const float* prev_clip,
                    float delta_time, float* rgb_out) {
    for (uint32_t i = 0; i < n; ++i) {
        const float* p = pos + 4 * (size_t)i;
        float pw[4], c[4], cp[4];
        mat4_point(model, p[0], p[1], p[2], pw);
        mat4_point(clip, pw[0], pw[1], pw[2], c);
        mat4_point(prev_clip, pw[0], pw[1], pw[2], cp);
        const float mvx = (c[0] / c[3] - cp[0] / cp[3]) * 0.5f;
        const float mvy = (c[1] / c[3] - cp[1] / cp[3]) * -0.5f;
        const float fx = mvx / delta_time, fy = mvy / delta_time;
        const float radius = std::sqrt(fx * fx + fy * fy);
        float angle = det_atan2(fy, fx);
        if (angle < 0.0f) angle = angle + PI_2_F;
        hsv_to_rgb(angle, std::fmin(std::fmax(radius, 0.0f), 1.0f), 1.0f, rgb_out + 3 * (size_t)i);
    }
}

}  // extern "C"
