// zb_device.cuh -- device-side scalar semantics shared by every kernel.  Each helper names the
// reference behaviour it has to reproduce (paths under arrufat/zignal src/).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace zb {

// border.zig:46-63 resolveIndex; -1 == null (contributes zero).  32-bit on the device: image axes
// are u32 and kernel offsets are small, so idx always fits.
__device__ __forceinline__ int resolve_index(int idx, int length, int border) {
    if (idx >= 0 && idx < length) return idx;
    if (border == 0 /*zero*/) return -1;
    if (length <= 0) return -1;
    if (border == 1 /*replicate*/) return idx < 0 ? 0 : length - 1;
    if (border == 2 /*mirror: reflect-101, period 2(n-1)*/) {
        if (length == 1) return 0;
        const int period = 2 * (length - 1);
        int m = idx % period;
        if (m < 0) m += period;
        return m >= length ? period - m : m;
    }
    /*wrap: floored modulo*/
    int m = idx % length;
    if (m < 0) m += length;
    return m;
}

// 64-bit variant for sampler coordinates that come from floats (interpolation.zig:314-322).
__device__ __forceinline__ long long resolve_index64(long long idx, long long length, int border) {
    if (idx >= 0 && idx < length) return idx;
    if (border == 0) return -1;
    if (length <= 0) return -1;
    if (border == 1) return idx < 0 ? 0 : length - 1;
    if (border == 2) {
        if (length == 1) return 0;
        const long long period = 2 * (length - 1);
        long long m = idx % period;
        if (m < 0) m += period;
        return m >= length ? period - m : m;
    }
    long long m = idx % length;
    if (m < 0) m += length;
    return m;
}

// meta.zig:121-128 clamp(u8, f32): round half away from zero, saturate; NaN -> 255 (Zig @min/@max
// return the non-NaN operand: @max(0, @min(NaN, 255)) == 255).
__device__ __forceinline__ uint8_t clamp_u8_from_float(float v) {
    if (v != v) return 255;
    const float r = roundf(v);  // half away from zero, exact in f32 (f64 widening in the reference changes nothing)
    return (uint8_t)fminf(fmaxf(r, 0.0f), 255.0f);
}

// std.math.clamp(v, 0, 1) = @max(0, @min(v, 1)); Zig's @min / @max return the non-NaN operand, so NaN gives 1 (255 once scaled
// to u8).  The reference's @max lowers to maxnum, which leaves the sign of a zero open: -0 gives +0 here and in the oracle.
// Written as two compares: nvcc folds fmaxf(0, fminf(v, 1)) into a saturating add (FADD.SAT), which gives 0 for NaN.  Every
// [0, 1] clamp of a float on the device goes through these two.
__device__ __forceinline__ float clamp01(float v) { return v < 1.0f ? (v > 0.0f ? v : 0.0f) : 1.0f; }
__device__ __forceinline__ double clamp01(double v) { return v < 1.0 ? (v > 0.0 ? v : 0.0) : 1.0; }

// convolution.zig:18-22 divClampU8: symmetric round-half-away divide, then clamp to u8.
template <typename Acc>
__device__ __forceinline__ uint8_t div_clamp_u8(Acc accum, Acc scale) {
    const Acc half = scale / 2;
    const Acc rounded = (accum + (accum >= 0 ? half : -half)) / scale;  // '/' truncates like @divTrunc
    return (uint8_t)(rounded < 0 ? 0 : (rounded > 255 ? 255 : rounded));
}

// Unfused f32 multiply-add in the reference's order (Zig never contracts a*b+c on this path).
__device__ __forceinline__ float mul_add_unfused(float a, float b, float acc) { return __fadd_rn(acc, __fmul_rn(a, b)); }

}  // namespace zb
