// zb_motion.cu -- Image.motionBlur (SURVEY 8(f).1; reference image.zig -> image/motion_blur.zig:65-436).
//   linear, horizontal / vertical  a uniform 1-D kernel through convolveSeparable with .replicate (:80-114) -> the fused / tile kernels;
//   linear, any other angle        per pixel a line integral of bilinear samples (:115-250);
//   radial zoom / spin             per pixel 8..32 bilinear samples along the ray / the arc through it (:252-436).
// The gathers are one thread per pixel: sample positions are computed once and shared by the channels (the reference recomputes the
// same f32 values per field), every product and sum is separately rounded in the reference's order, so linear and zoom are
// bit-exact; spin calls atan2f / cosf / sinf per sample, whose last bit differs between libms (checked at 1e-5 / one 8-bit step).
#include <cmath>
#include <vector>

#include "zb_conv.h"
#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {

int conv_separable_dispatch(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny, int border,
                            cudaStream_t s, int row0, int row1);   // zb_api_conv.cu

namespace {

struct MotionParams {
    const void* src;
    void* dst;
    size_t src_stride, dst_stride;   // pixels
    int rows, cols;
    // linear
    float cos_a, sin_a, half_dist;
    unsigned loop_limit;
    // radial
    float cx, cy, clamped, max_distance;
    int num_samples, spin;
};

template <typename CT, int CH>
__device__ __forceinline__ float comp(const MotionParams& p, int r, int c, int k) {
    return (float)((const CT*)p.src)[((size_t)r * p.src_stride + c) * CH + k];
}

// motion_blur.zig:135-152 / :316-333: bilinear tap with x1 / y1 clamped to the last column / row; adds to sum[] per channel.
template <typename CT, int CH>
__device__ __forceinline__ void tap(const MotionParams& p, float sx, float sy, float (&sum)[CH]) {
    const int x0 = (int)floorf(sx), y0 = (int)floorf(sy);
    const int x1 = min(x0 + 1, p.cols - 1), y1 = min(y0 + 1, p.rows - 1);
    const float fx = __fsub_rn(sx, (float)x0), fy = __fsub_rn(sy, (float)y0);
    const float gx = __fsub_rn(1.0f, fx), gy = __fsub_rn(1.0f, fy);
#pragma unroll
    for (int k = 0; k < CH; ++k) {
        const float v00 = comp<CT, CH>(p, y0, x0, k), v10 = comp<CT, CH>(p, y0, x1, k), v01 = comp<CT, CH>(p, y1, x0, k),
                    v11 = comp<CT, CH>(p, y1, x1, k);
        const float v0 = __fadd_rn(__fmul_rn(v00, gx), __fmul_rn(v10, fx));
        const float v1 = __fadd_rn(__fmul_rn(v01, gx), __fmul_rn(v11, fx));
        sum[k] = __fadd_rn(sum[k], __fadd_rn(__fmul_rn(v0, gy), __fmul_rn(v1, fy)));
    }
}

template <typename CT, int CH>
__device__ __forceinline__ void finish(const MotionParams& p, int r, int c, const float (&sum)[CH], float count) {
#pragma unroll
    for (int k = 0; k < CH; ++k) {
        const float result = count > 0.0f ? __fdiv_rn(sum[k], count) : comp<CT, CH>(p, r, c, k);       // :158, :346
        CT* out = (CT*)p.dst + ((size_t)r * p.dst_stride + c) * CH + k;
        if constexpr (sizeof(CT) == 1) *out = (uint8_t)truncf(fmaxf(0.0f, fminf(255.0f, roundf(result))));   // :160
        else *out = result;
    }
}

template <typename CT, int CH>
__global__ void __launch_bounds__(256) motion_line_kernel(const MotionParams p) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31), r = ZB_GRID_ROW() * 8 + (threadIdx.x >> 5);
    if (c >= p.cols || r >= p.rows) return;
    const float fcols = (float)p.cols, frows = (float)p.rows;
    float sum[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) sum[k] = 0.0f;
    float count = 0.0f, t = -p.half_dist;
    for (unsigned it = 0; it < p.loop_limit; ++it) {                  // :125-156
        if (t > p.half_dist) break;
        const float sx = __fadd_rn((float)c, __fmul_rn(t, p.cos_a)), sy = __fadd_rn((float)r, __fmul_rn(t, p.sin_a));
        if (sx >= 0.0f && sx < fcols && sy >= 0.0f && sy < frows) {
            tap<CT, CH>(p, sx, sy, sum);
            count = __fadd_rn(count, 1.0f);
        }
        t = __fadd_rn(t, 1.0f);
    }
    finish<CT, CH>(p, r, c, sum, count);
}

template <typename CT, int CH>
__global__ void __launch_bounds__(256) motion_radial_kernel(const MotionParams p) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31), r = ZB_GRID_ROW() * 8 + (threadIdx.x >> 5);
    if (c >= p.cols || r >= p.rows) return;
    const float fcols = (float)p.cols, frows = (float)p.rows;
    const float dx = __fsub_rn((float)c, p.cx), dy = __fsub_rn((float)r, p.cy);
    const float distance = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));                 // :287
    const float blur_amount = p.spin ? __fmul_rn(p.clamped, 0.5f)
                                     : __fmul_rn(__fmul_rn(__fdiv_rn(distance, p.max_distance), p.clamped), 20.0f);   // :294-297
    const float angle = p.spin ? atan2f(dy, dx) : 0.0f;
    const float n1 = (float)(p.num_samples - 1);
    float sum[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) sum[k] = 0.0f;
    int count = 0;
    for (int s = 0; s < p.num_samples; ++s) {
        const float t = __fdiv_rn(__fsub_rn((float)s, __fdiv_rn(n1, 2.0f)), n1);                        // :304
        float sx, sy;
        if (!p.spin) {
            const float scale = __fadd_rn(1.0f, __fmul_rn(__fmul_rn(t, blur_amount), 0.1f));            // :310-313
            sx = __fadd_rn(p.cx, __fmul_rn(dx, scale));
            sy = __fadd_rn(p.cy, __fmul_rn(dy, scale));
        } else {
            const float new_angle = __fadd_rn(angle, __fmul_rn(t, blur_amount));                        // :315-319
            sx = __fadd_rn(p.cx, __fmul_rn(distance, cosf(new_angle)));
            sy = __fadd_rn(p.cy, __fmul_rn(distance, sinf(new_angle)));
        }
        if (sx >= 0.0f && sx < fcols && sy >= 0.0f && sy < frows) {
            tap<CT, CH>(p, sx, sy, sum);
            ++count;
        }
    }
    finish<CT, CH>(p, r, c, sum, (float)count);
}

template <bool RADIAL>
int launch(const MotionParams& p, int pixfmt, cudaStream_t s) {
    const dim3 grid = row_grid(div_up(p.cols, 32), div_up(p.rows, 8));
#define ZB_MOTION_CASE(CT, CH)                                                  \
    if (RADIAL) motion_radial_kernel<CT, CH><<<grid, 256, 0, s>>>(p);           \
    else motion_line_kernel<CT, CH><<<grid, 256, 0, s>>>(p);                    \
    break
    switch (pixfmt) {
        case ZB_PIX_U8: ZB_MOTION_CASE(uint8_t, 1);
        case ZB_PIX_F32: ZB_MOTION_CASE(float, 1);
        case ZB_PIX_RGB8: ZB_MOTION_CASE(uint8_t, 3);
        case ZB_PIX_RGBA8: ZB_MOTION_CASE(uint8_t, 4);
        case ZB_PIX_RGBAF32: ZB_MOTION_CASE(float, 4);
        default: return ZB_ERR_UNSUPPORTED;
    }
#undef ZB_MOTION_CASE
    ZB_LAUNCHED();
    return ZB_OK;
}

int check_images(const zb_image* src, const zb_image* dst, int pixfmt) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;
    return ZB_OK;
}

MotionParams base_params(const zb_image* src, zb_image* dst) {
    MotionParams p{};
    p.src = src->data;
    p.dst = dst->data;
    p.src_stride = src->stride;
    p.dst_stride = dst->stride;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    return p;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_motion_blur_linear(const zb_image* src, zb_image* dst, int pixfmt, float angle, float cos_a, float sin_a, uint32_t distance,
                                     zb_stream stream) {
    (void)angle;
    int rc = check_images(src, dst, pixfmt);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (distance == 0) return zb_copy(src, dst, pixfmt, stream);                                        // :66-69
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    const float epsilon = 0.001f;                                                                       // :77-79
    const bool horizontal = std::fabs(sin_a) < epsilon, vertical = std::fabs(cos_a) < epsilon;
    if (horizontal || vertical) {
        if (distance > (uint32_t)kMaxTaps) return ZB_ERR_UNSUPPORTED;
        std::vector<float> kernel(distance, 1.0f / (float)distance);                                    // :88-91
        const float identity[1] = {1.0f};
        return horizontal ? conv_separable_dispatch(src, dst, pixfmt, kernel.data(), (int)distance, identity, 1, ZB_BORDER_REPLICATE, s, 0, -1)
                          : conv_separable_dispatch(src, dst, pixfmt, identity, 1, kernel.data(), (int)distance, ZB_BORDER_REPLICATE, s, 0, -1);
    }
    if (images_overlap(src, dst, pixel_bytes(pixfmt))) return ZB_ERR_INVALID_ARGUMENT;     // a gather: the reference reads `image` while it writes `out`
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;
    MotionParams p = base_params(src, dst);
    p.cos_a = cos_a;
    p.sin_a = sin_a;
    p.half_dist = (float)distance / 2.0f;                                                               // :74
    p.loop_limit = distance > 0xfffffffdu ? 0xffffffffu : distance + 2;                                 // :123
    if ((rc = launch<false>(p, pixfmt, s))) return rc;
    t_last_kernel = "motion_line";
    return ZB_OK;
}

extern "C" int zb_motion_blur_radial(const zb_image* src, zb_image* dst, int pixfmt, float center_x, float center_y, float strength, int spin,
                                     zb_stream stream) {
    int rc = check_images(src, dst, pixfmt);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    if (strength == 0) return zb_copy(src, dst, pixfmt, stream);                                        // :262-265
    if (images_overlap(src, dst, pixel_bytes(pixfmt))) return ZB_ERR_INVALID_ARGUMENT;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;
    MotionParams p = base_params(src, dst);
    p.cx = center_x * (float)(src->cols - 1);                                                           // :268-269
    p.cy = center_y * (float)(src->rows - 1);
    p.clamped = std::fmax(0.0f, std::fmin(1.0f, strength));                                             // :272
    p.num_samples = 8 + (int)std::trunc(p.clamped * 24.0f);                                             // :275-277
    p.max_distance = std::sqrt(p.cx * p.cx + p.cy * p.cy);                                              // :293
    p.spin = spin ? 1 : 0;
    if ((rc = launch<true>(p, pixfmt, s))) return rc;
    t_last_kernel = spin ? "motion_spin" : "motion_zoom";
    return ZB_OK;
}
