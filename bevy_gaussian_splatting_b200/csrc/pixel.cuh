// pixel.cuh -- the frame's pixel encoder: one pixel's blended state (premultiplied rgb C, transmittance T) -> the target,
// in each format and output mode.  The blend kernels (raster.cu) and the shutter resolve (shutter.cu) write every frame
// pixel through write_pixel, so a resolved frame is encoded exactly as a blended one.  Both files are built alike
// (csrc/Makefile), so the encoder's arithmetic compiles to the same instructions in each.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace bgs {

__device__ __forceinline__ float linear_to_srgb(float c) {
    c = fminf(fmaxf(c, 0.0f), 1.0f);
    // __powf = ex2.approx(lg2.approx(c) / 2.4): ~1e-6 relative, far below the 8-bit quantisation step (the full
    // powf was 7 % of the kernel's instructions)
    return c <= 0.0031308f ? 12.92f * c : 1.055f * __powf(c, 1.0f / 2.4f) - 0.055f;
}

// ---- frame output.  `format` = BGS_FORMAT_* | output mode << 8:
//   mode 0: the splat layer over an opaque black clear (examples/headless.rs:70): (C, 1)
//   mode 1 (BGS_FLAG_PREMULTIPLIED_OUT): the layer alone, premultiplied: (C, 1 - T)
//   mode 2 (BGS_FLAG_BLEND_OVER_TARGET): blended over what the target holds, dst = src + (1 - src.a) dst on all four
//           channels (PREMULTIPLIED_ALPHA_BLENDING, render/mod.rs:944-948): (C + T dst.rgb, (1 - T) + T dst.a)
constexpr uint32_t OUT_PREMUL = 1u, OUT_OVER = 2u;
__device__ __forceinline__ float srgb_decode(float c) {
    return c <= 0.04045f ? c * (1.0f / 12.92f) : __powf((c + 0.055f) * (1.0f / 1.055f), 2.4f);
}
__device__ __forceinline__ float4 read_pixel(const void* out, uint32_t fmt, size_t pix) {
    if (fmt == BGS_FORMAT_RGBA32F) return reinterpret_cast<const float4*>(out)[pix];
    if (fmt == BGS_FORMAT_RGBA16F) {
        const uint2 v = reinterpret_cast<const uint2*>(out)[pix];
        const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), hi = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
        return make_float4(lo.x, lo.y, hi.x, hi.y);
    }
    const uint32_t v = reinterpret_cast<const uint32_t*>(out)[pix];
    return make_float4(srgb_decode((float)(v & 255u) * (1.0f / 255.0f)), srgb_decode((float)((v >> 8) & 255u) * (1.0f / 255.0f)),
                       srgb_decode((float)((v >> 16) & 255u) * (1.0f / 255.0f)), (float)(v >> 24) * (1.0f / 255.0f));
}
// pixel encoders: RGBA16F, and sRGB8 with a linear alpha byte (or 255 when !with_alpha)
__device__ __forceinline__ uint2 pack_rgba16f(float r, float g, float b, float a) {
    const __half2 lo = __floats2half2_rn(r, g), hi = __floats2half2_rn(b, a);
    return make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
}
__device__ __forceinline__ uint32_t pack_srgb8(float r, float g, float b, float a, bool with_alpha) {
    const uint32_t r8 = (uint32_t)(linear_to_srgb(r) * 255.0f + 0.5f);
    const uint32_t g8 = (uint32_t)(linear_to_srgb(g) * 255.0f + 0.5f);
    const uint32_t b8 = (uint32_t)(linear_to_srgb(b) * 255.0f + 0.5f);
    const uint32_t a8 = with_alpha ? (uint32_t)(fminf(fmaxf(a, 0.0f), 1.0f) * 255.0f + 0.5f) : 255u;
    return r8 | (g8 << 8) | (b8 << 16) | (a8 << 24);
}
// one pixel's accumulated premultiplied colour (r, g, b) and remaining transmittance T -> the frame
__device__ __forceinline__ void write_pixel(void* out, uint32_t format, size_t pix, float r, float g, float b, float T) {
    const uint32_t fmt = format & 0xFFu, mode = format >> 8;
    float a = 1.0f;
    if (mode & OUT_OVER) {
        const float4 d = read_pixel(out, fmt, pix);
        r = fmaf(T, d.x, r); g = fmaf(T, d.y, g); b = fmaf(T, d.z, b);
        a = fmaf(T, d.w, 1.0f - T);
    } else if (mode & OUT_PREMUL) {
        a = 1.0f - T;
    }
    if (fmt == BGS_FORMAT_RGBA32F) {
        reinterpret_cast<float4*>(out)[pix] = make_float4(r, g, b, a);
    } else if (fmt == BGS_FORMAT_RGBA16F) {
        reinterpret_cast<uint2*>(out)[pix] = pack_rgba16f(r, g, b, a);
    } else {
        reinterpret_cast<uint32_t*>(out)[pix] = pack_srgb8(r, g, b, a, mode != 0);
    }
}

}  // namespace bgs
