// zb_blend.cuh -- Rgba(u8).blend(overlay, mode) = blendColors(u8, base, overlay, mode) (reference blending.zig:26-156) for the
// samplers that composite instead of assigning (Image.insert with a blend mode, image.zig:67-95 assignPixel).  f32 arithmetic in
// the reference's operation order, every product and sum separately rounded (Zig never contracts), so results match bit for bit.
#pragma once
#include "zb_device.cuh"

namespace zb {

__device__ __forceinline__ float blend_channel(float bv, float ov, int mode) {
    const float one_b = __fsub_rn(1.0f, bv), one_o = __fsub_rn(1.0f, ov);
    switch (mode) {
        case ZB_BLEND_NORMAL: return ov;
        case ZB_BLEND_MULTIPLY: return __fmul_rn(bv, ov);
        case ZB_BLEND_SCREEN: return __fsub_rn(1.0f, __fmul_rn(one_b, one_o));
        case ZB_BLEND_OVERLAY:
            return bv < 0.5f ? __fmul_rn(__fmul_rn(2.0f, bv), ov) : __fsub_rn(1.0f, __fmul_rn(__fmul_rn(2.0f, one_b), one_o));
        case ZB_BLEND_SOFT_LIGHT:
            return ov <= 0.5f ? __fsub_rn(bv, __fmul_rn(__fmul_rn(__fsub_rn(1.0f, __fmul_rn(2.0f, ov)), bv), one_b))
                              : __fadd_rn(bv, __fmul_rn(__fsub_rn(__fmul_rn(2.0f, ov), 1.0f), __fsub_rn(__fsqrt_rn(bv), bv)));
        case ZB_BLEND_HARD_LIGHT:
            return ov < 0.5f ? __fmul_rn(__fmul_rn(2.0f, ov), bv) : __fsub_rn(1.0f, __fmul_rn(__fmul_rn(2.0f, one_o), one_b));
        case ZB_BLEND_COLOR_DODGE: return bv == 0.0f ? 0.0f : (ov >= 1.0f ? 1.0f : fminf(1.0f, __fdiv_rn(bv, one_o)));
        case ZB_BLEND_COLOR_BURN: return bv >= 1.0f ? 1.0f : (ov <= 0.0f ? 0.0f : fmaxf(0.0f, __fsub_rn(1.0f, __fdiv_rn(one_b, ov))));
        case ZB_BLEND_DARKEN: return fminf(bv, ov);
        case ZB_BLEND_LIGHTEN: return fmaxf(bv, ov);
        case ZB_BLEND_DIFFERENCE: return fabsf(__fsub_rn(bv, ov));
        default: return __fsub_rn(__fadd_rn(bv, ov), __fmul_rn(__fmul_rn(2.0f, bv), ov));   // exclusion
    }
}

// Pixels as little-endian packed words: r | g << 8 | b << 16 | a << 24 (the memory layout of Rgba(u8)).
__device__ __forceinline__ uint32_t blend_rgba8(uint32_t base, uint32_t overlay, int mode) {
    if (mode == ZB_BLEND_NONE) return overlay;                                    // :27
    const uint32_t oa = overlay >> 24, ba = base >> 24;
    if (oa == 0) return base;                                                     // :30
    if (ba == 0) return overlay;                                                  // :33
    if (mode == ZB_BLEND_NORMAL && oa == 255) return overlay;                     // :36
    float b[4], o[4], out[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {                                                 // color.zig:484-494 as(f32): v / 255
        b[k] = __fdiv_rn((float)((base >> (8 * k)) & 255u), 255.0f);
        o[k] = __fdiv_rn((float)((overlay >> (8 * k)) & 255u), 255.0f);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = blend_channel(b[k], o[k], mode);
    if (oa == 255) {                                                              // :127-136
        out[3] = 1.0f;
    } else {                                                                      // :137-154
        const float base_weight = __fmul_rn(b[3], __fsub_rn(1.0f, o[3]));
        const float result_a = __fadd_rn(o[3], base_weight);
        if (result_a <= 0.0f) return 0u;
        const float inv_result_a = __fdiv_rn(1.0f, result_a);
#pragma unroll
        for (int k = 0; k < 3; ++k) out[k] = __fmul_rn(__fadd_rn(__fmul_rn(out[k], o[3]), __fmul_rn(b[k], base_weight)), inv_result_a);
        out[3] = result_a;
    }
    uint32_t res = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {                                                 // color.zig:496-501 as(u8): @round(255 * clamp(v, 0, 1))
        res |= (uint32_t)roundf(__fmul_rn(255.0f, clamp01(out[k]))) << (8 * k);
    }
    return res;
}

}  // namespace zb
