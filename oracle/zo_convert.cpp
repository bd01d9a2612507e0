// zo_convert.cpp -- CPU oracle (TEST INFRASTRUCTURE ONLY, see zignal_oracle.h) for Image.convert / convertInto (reference image.zig:396-421):
// per pixel convertColor(TargetType, px) (color.zig:108-151) between the five pixel types of the path -- u8, f32, Rgb(u8), Rgba(u8),
// Rgba(f32).  Each branch names the rule of convertColor it restates.
#include "zo_common.h"

namespace zo {
namespace {

// std.math.clamp(v, 0, 1) = @max(0, @min(v, 1)): NaN gives 1 (@min returns the non-NaN operand).  -0 gives +0, as on the device: the
// reference's @max lowers to maxnum, which leaves the sign of a zero open, so both sides pin +0.
inline float clamp01(float v) { return v < 1.0f ? (v > 0.0f ? v : 0.0f) : 1.0f; }
// Gray / Rgb / Rgba .as(u8) from a float component: @round(255 * clamp(v, 0, 1)) in that float type (color.zig:376-379, 496-501, 553)
inline uint8_t unit_to_u8(float v) { return (uint8_t)std::round(255.0f * clamp01(v)); }
// .as(f32) from a u8 component: @as(f32, v) / 255 (color.zig:369-373, 488-493, 550)
inline float u8_to_unit(uint8_t v) { return (float)v / 255.0f; }
// rgbToGray(u8) (color.zig:1031-1041)
inline uint8_t luma_u8(uint8_t r, uint8_t g, uint8_t b) {
    const int y = (13933 * (int)r + 46871 * (int)g + 4732 * (int)b + 32768) >> 16;
    return (uint8_t)(y < 0 ? 0 : (y > 255 ? 255 : y));
}
// rgbToGray(f32) (color.zig:1043-1045): clamp(luma_r * r + luma_g * g + luma_b * b, 0, 1), coefficients rounded to f32
inline float luma_f32(float r, float g, float b) { return clamp01(0.2126f * r + 0.7152f * g + 0.0722f * b); }

struct Px {            // one pixel of any of the five formats, components as stored
    uint8_t u[4];
    float f[4];
};

inline void load(const zo_image* im, int fmt, size_t r, size_t c, Px& p) {
    const size_t i = r * (size_t)im->stride + c;
    switch (fmt) {
        case ZO_PIX_U8: p.u[0] = ((const uint8_t*)im->data)[i]; break;
        case ZO_PIX_F32: p.f[0] = ((const float*)im->data)[i]; break;
        case ZO_PIX_RGB8: for (int k = 0; k < 3; ++k) p.u[k] = ((const uint8_t*)im->data)[i * 3 + k]; break;
        case ZO_PIX_RGBA8: for (int k = 0; k < 4; ++k) p.u[k] = ((const uint8_t*)im->data)[i * 4 + k]; break;
        default: for (int k = 0; k < 4; ++k) p.f[k] = ((const float*)im->data)[i * 4 + k]; break;
    }
}
inline void store(zo_image* im, int fmt, size_t r, size_t c, const Px& p) {
    const size_t i = r * (size_t)im->stride + c;
    switch (fmt) {
        case ZO_PIX_U8: ((uint8_t*)im->data)[i] = p.u[0]; break;
        case ZO_PIX_F32: ((float*)im->data)[i] = p.f[0]; break;
        case ZO_PIX_RGB8: for (int k = 0; k < 3; ++k) ((uint8_t*)im->data)[i * 3 + k] = p.u[k]; break;
        case ZO_PIX_RGBA8: for (int k = 0; k < 4; ++k) ((uint8_t*)im->data)[i * 4 + k] = p.u[k]; break;
        default: for (int k = 0; k < 4; ++k) ((float*)im->data)[i * 4 + k] = p.f[k]; break;
    }
}

// convertColor(Dst, src) for src != dst
void convert_px(int sf, int df, const Px& s, Px& d) {
    const bool s_scalar = sf == ZO_PIX_U8 || sf == ZO_PIX_F32, d_scalar = df == ZO_PIX_U8 || df == ZO_PIX_F32;
    if (s_scalar && d_scalar) {                                              // color.zig:113-118 scalar <-> scalar
        if (sf == ZO_PIX_U8) d.f[0] = (float)s.u[0] / 255.0f;
        else {
            double v = (double)s.f[0];
            v = zig_max(0.0, zig_min(v, 1.0));   // std.math.clamp: NaN -> 1
            d.u[0] = (uint8_t)std::round(v * 255.0);                         // through f64 (:116-117)
        }
        return;
    }
    if (s_scalar) {                                                          // :121-131 scalar -> color: Gray{y}.as(DestT).to(space)
        if (df == ZO_PIX_RGBAF32) {
            const float y = sf == ZO_PIX_U8 ? u8_to_unit(s.u[0]) : s.f[0];
            d.f[0] = d.f[1] = d.f[2] = y;
            d.f[3] = 1.0f;                                                   // Rgb.to(.rgba): alpha 1.0 (:355)
        } else {
            const uint8_t y = sf == ZO_PIX_U8 ? s.u[0] : unit_to_u8(s.f[0]);
            d.u[0] = d.u[1] = d.u[2] = y;
            d.u[3] = 255;
        }
        return;
    }
    if (d_scalar) {                                                          // :133-136 color -> scalar: source.to(.gray).as(Dest).y
        if (sf == ZO_PIX_RGBAF32) {
            const float y = luma_f32(s.f[0], s.f[1], s.f[2]);                // Rgba.to(.rgb).to(.gray), alpha dropped (:477-479)
            if (df == ZO_PIX_F32) d.f[0] = y; else d.u[0] = unit_to_u8(y);
        } else {
            const uint8_t y = luma_u8(s.u[0], s.u[1], s.u[2]);
            if (df == ZO_PIX_U8) d.u[0] = y; else d.f[0] = u8_to_unit(y);
        }
        return;
    }
    // :138-150 color -> color
    if (df == ZO_PIX_RGBAF32) {                                              // source.as(f32).to(.rgba)
        for (int k = 0; k < 3; ++k) d.f[k] = u8_to_unit(s.u[k]);
        d.f[3] = sf == ZO_PIX_RGBA8 ? u8_to_unit(s.u[3]) : 1.0f;
    } else if (sf == ZO_PIX_RGBAF32) {                                       // source.to(space).as(u8)
        for (int k = 0; k < 3; ++k) d.u[k] = unit_to_u8(s.f[k]);
        d.u[3] = unit_to_u8(s.f[3]);                                         // only stored for Rgba(u8)
    } else {                                                                 // Rgb(u8) <-> Rgba(u8)
        for (int k = 0; k < 3; ++k) d.u[k] = s.u[k];
        d.u[3] = 255;
    }
}

}  // namespace
}  // namespace zo

extern "C" int zo_convert(const zo_image* src, int src_pixfmt, zo_image* dst, int dst_pixfmt) {
    using namespace zo;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;    // image.zig:397 assert(hasSameShape)
    if (src_pixfmt < ZO_PIX_U8 || src_pixfmt > ZO_PIX_RGBAF32 || dst_pixfmt < ZO_PIX_U8 || dst_pixfmt > ZO_PIX_RGBAF32) return ZO_ERR_UNSUPPORTED;
    for (size_t r = 0; r < src->rows; ++r)
        for (size_t c = 0; c < src->cols; ++c) {
            Px s{}, d{};
            load(src, src_pixfmt, r, c, s);
            if (src_pixfmt == dst_pixfmt) d = s; else convert_px(src_pixfmt, dst_pixfmt, s, d);
            store(dst, dst_pixfmt, r, c, d);
        }
    return ZO_OK;
}
