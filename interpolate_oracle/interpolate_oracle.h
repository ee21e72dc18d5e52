/*
 * interpolate_oracle.h -- CPU ORACLE of the interpolation (src/morph/interpolate.wgsl:51-119, the reference's
 * GaussianInterpolate { lhs, rhs }).  TEST INFRASTRUCTURE ONLY: the product (libbgs.so) never links, loads or calls it.
 * Built beside oracle/ (the render oracle) by __graft_entry__.build().
 *
 * The rule (include/bgs.h, bgs_cloud_interpolate), one scalar restatement per gaussian and lane, every operation f32
 * round-to-nearest-even without FMA (-ffp-contract=off), subnormals kept:
 *   t: d = time_stop - time_start; |d| < 1e-6f ? (time >= time_stop ? 1 : 0) : min(max((time - time_start) / d, 0), 1);
 *   each lane mix(a, b, t) = a*(1-t) + b*t; the rotation (w, x, y, z) normalised: l2 = ((w*w + x*x) + y*y) + z*z,
 *   l2 <= 0 -> (0, 0, 0, 1), else each lane / sqrt(l2);
 *   f16 halves widened exactly, narrowed round-to-nearest-even (+-inf past the range); the covariance record's fourth
 *   word is opacity (high half) | +0 (low half).
 *
 * Planes are the arrays the upload calls take and the download calls return: planes[0] = pos_vis (n*4 f32),
 * planes[1] = sh (f32: n*48 f32; f16 layouts: n*24 u32), planes[2] = rotation (f32: n*4 f32) or the second plane
 * (f16 layouts: n*4 u32), planes[3] = scale_opacity (f32 layout only, n*4 f32).
 */
#ifndef INTERPOLATE_ORACLE_H
#define INTERPOLATE_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

enum { ORC_INTERP_F32 = 0, ORC_INTERP_F16 = 1, ORC_INTERP_F16_COV = 2 };

/* 0 and *t = the factor; -1 (t untouched) when an input is not finite or the factor is NaN (what libbgs refuses) */
int orc_interp_factor(float time, float time_start, float time_stop, float* t);
/* out := mix(lhs, rhs, t) over n gaussians of one layout */
void orc_interp(uint32_t n, int layout, float t, const void* const lhs[4], const void* const rhs[4], void* const out[4]);
/* the f16 conversions the f16 layouts use */
float orc_half_to_float(uint16_t h);
uint16_t orc_float_to_half(float f);

#ifdef __cplusplus
}
#endif
#endif
