// zb_convert.cuh -- convertColor(TargetType, pixel) (reference color.zig:108-151) for one pixel, on the device: the rules of
// Image.convert (zb_convert.cu) as a function, also used by the mixed-type Image.insert (zb_insert_mixed.cu, image.zig:67-95).
#pragma once
#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {

__device__ __forceinline__ uint8_t unit_to_u8(float v) { return (uint8_t)roundf(__fmul_rn(255.0f, clamp01(v))); }
__device__ __forceinline__ float u8_to_unit(uint8_t v) { return __fdiv_rn((float)v, 255.0f); }
__device__ __forceinline__ uint8_t luma_u8(uint8_t r, uint8_t g, uint8_t b) {
    const int y = (13933 * (int)r + 46871 * (int)g + 4732 * (int)b + 32768) >> 16;
    return (uint8_t)min(max(y, 0), 255);
}
// rgbToGray(f32) before its clamp
__device__ __forceinline__ float luma_sum_f32(float r, float g, float b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(0.2126f, r), __fmul_rn(0.7152f, g)), __fmul_rn(0.0722f, b));
}
__device__ __forceinline__ float luma_f32(float r, float g, float b) { return clamp01(luma_sum_f32(r, g, b)); }

template <int FMT> struct Fmt;
template <> struct Fmt<ZB_PIX_U8> { using CT = uint8_t; static constexpr int N = 1; };
template <> struct Fmt<ZB_PIX_F32> { using CT = float; static constexpr int N = 1; };
template <> struct Fmt<ZB_PIX_RGB8> { using CT = uint8_t; static constexpr int N = 3; };
template <> struct Fmt<ZB_PIX_RGBA8> { using CT = uint8_t; static constexpr int N = 4; };
template <> struct Fmt<ZB_PIX_RGBAF32> { using CT = float; static constexpr int N = 4; };

// s: S::N components of the source format, d: D::N components of the destination format (SF != DF)
template <int SF, int DF>
__device__ __forceinline__ void convert_color(const typename Fmt<SF>::CT* s, typename Fmt<DF>::CT* d) {
    using S = Fmt<SF>;
    using D = Fmt<DF>;
    constexpr bool s_float = sizeof(typename S::CT) == 4, d_float = sizeof(typename D::CT) == 4;
    if constexpr (S::N == 1 && D::N == 1) {                       // scalar <-> scalar, color.zig:113-118
        if constexpr (!s_float) {
            d[0] = __fdiv_rn((float)s[0], 255.0f);
        } else {
            d[0] = (uint8_t)round(clamp01((double)s[0]) * 255.0);   // through f64
        }
    } else if constexpr (S::N == 1) {                             // scalar -> colour, :121-131
        if constexpr (d_float) {
            float y;
            if constexpr (s_float) y = s[0]; else y = u8_to_unit(s[0]);
            d[0] = d[1] = d[2] = y;
            d[3] = 1.0f;
        } else {
            uint8_t y;
            if constexpr (s_float) y = unit_to_u8(s[0]); else y = s[0];
            d[0] = d[1] = d[2] = y;
            if constexpr (D::N == 4) d[3] = 255;
        }
    } else if constexpr (D::N == 1) {                             // colour -> scalar, :133-136
        if constexpr (s_float) {
            const float y = luma_f32(s[0], s[1], s[2]);
            if constexpr (d_float) d[0] = y; else d[0] = unit_to_u8(y);
        } else {
            const uint8_t y = luma_u8(s[0], s[1], s[2]);
            if constexpr (d_float) d[0] = u8_to_unit(y); else d[0] = y;
        }
    } else if constexpr (d_float) {                               // 8-bit colour -> Rgba(f32): source.as(f32).to(.rgba), :144-148
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = u8_to_unit(s[k]);
        if constexpr (S::N == 4) d[3] = u8_to_unit(s[3]); else d[3] = 1.0f;
    } else if constexpr (s_float) {                               // Rgba(f32) -> 8-bit colour: source.to(space).as(u8), :150
#pragma unroll
        for (int k = 0; k < D::N; ++k) d[k] = unit_to_u8(s[k]);
    } else {                                                      // Rgb(u8) <-> Rgba(u8)
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = s[k];
        if constexpr (D::N == 4) d[3] = 255;
    }
}

}  // namespace zb
