// zb_color.cu -- Image.convertInto between the 33 colour formats (reference image.zig:396-421, color.zig:108-151): zb_convert_color.
// The host turns the (source, destination) pair into a ColorPlan: the `.as()` rules at both ends, the compute type, and the hops of
// the reference's `to` switches from one space to the other.  One elementwise kernel runs it, templated on the storage types of the
// two ends and the compute type (27 instances); the spaces are uniform arguments, so the pair costs no instantiation of its own.
#include "zb_color.cuh"
#include "zb_internal.h"

namespace zb {
namespace {

using namespace color;

constexpr int kComponentBytes[3] = {1, 4, 8};
static_assert(CU8 == ZB_COMPONENT_U8 && CF32 == ZB_COMPONENT_F32 && CF64 == ZB_COMPONENT_F64, "component numbering");
static_assert(SCALAR == ZB_SPACE_SCALAR && YCBCR == ZB_SPACE_YCBCR, "space numbering");

// The formats the reference allows: every space takes f32 and f64; u8 only the scalar, Gray, Rgb, Rgba and Ycbcr
// (color.zig:280-285, 394-399, 516-521, 925-930; the others compile-error on a non-float T).
bool valid_format(int space, int component) {
    if (space < 0 || space >= NSPACES || component < ZB_COMPONENT_U8 || component > ZB_COMPONENT_F64) return false;
    if (component != ZB_COMPONENT_U8) return true;
    return space == SCALAR || space == GRAY || space == RGB || space == RGBA || space == YCBCR;
}

// src and dst are not __restrict__: dst may be src itself (same pixel size, same view), where each pixel's components are read, then
// written, by the one thread that owns the pixel.
template <typename S, typename D, typename C>
__global__ void __launch_bounds__(256) color_kernel(ColorPlan p, const S* src, size_t src_stride, D* dst, size_t dst_stride, int rows,
                                                    int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = ZB_GRID_ROW();
    if (c >= cols || r >= rows) return;
    const S* sp = src + ((size_t)r * src_stride + c) * p.ns;
    D* dp = dst + ((size_t)r * dst_stride + c) * p.nd;
    S s[4] = {};
#pragma unroll
    for (int k = 0; k < 4; ++k) if (k < p.ns) s[k] = sp[k];
    D d[4];
    convert_pixel<S, D, C>(p, s, d);
#pragma unroll
    for (int k = 0; k < 4; ++k) if (k < p.nd) dp[k] = d[k];
}

template <typename F>
int dispatch_component(int k, F&& f) {
    switch (k) {
        case ZB_COMPONENT_U8: return f(std::integral_constant<int, ZB_COMPONENT_U8>{});
        case ZB_COMPONENT_F32: return f(std::integral_constant<int, ZB_COMPONENT_F32>{});
        case ZB_COMPONENT_F64: return f(std::integral_constant<int, ZB_COMPONENT_F64>{});
    }
    return ZB_ERR_UNSUPPORTED;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_convert_color(const zb_color_image* src, zb_color_image* dst, zb_stream stream) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (!valid_format(src->space, src->component) || !valid_format(dst->space, dst->component)) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;      // image.zig:397
    const size_t scb = kComponentBytes[src->component], dcb = kComponentBytes[dst->component];
    const size_t spb = scb * channels_of_space(src->space), dpb = dcb * channels_of_space(dst->space);
    if ((uintptr_t)src->data % scb || (uintptr_t)dst->data % dcb) return ZB_ERR_INVALID_ARGUMENT;
    const size_t rows = src->rows, cols = src->cols;
    const bool same_view = src->data == dst->data && src->stride == dst->stride && spb == dpb;
    if (rows && cols && !same_view && src->data && dst->data) {   // any other overlap would let one pixel's write reach another's read
        const uintptr_t a0 = (uintptr_t)src->data, a1 = a0 + ((rows - 1) * src->stride + cols) * spb;
        const uintptr_t b0 = (uintptr_t)dst->data, b1 = b0 + ((rows - 1) * dst->stride + cols) * dpb;
        if (a0 < b1 && b0 < a1) return ZB_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (src->space == dst->space && src->component == dst->component) {                         // :398-399
        if (same_view || rows == 0 || cols == 0) return ZB_OK;
        return span_copy(dst->data, dst->stride * dpb, src->data, src->stride * spb, cols * spb, rows, cudaMemcpyDeviceToDevice, s);
    }
    if (rows > 0x7fffffffu || cols * spb > 0x7fffffffu || cols * dpb > 0x7fffffffu) return ZB_ERR_UNSUPPORTED;
    if (rows == 0 || cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const ColorPlan plan = make_plan(src->space, src->component, dst->space, dst->component);
    const dim3 grid = row_grid(div_up(cols, 256), rows);
    rc = dispatch_component(src->component, [&](auto sk) -> int {
        return dispatch_component(dst->component, [&](auto dk) -> int {
            return dispatch_component(plan.compute, [&](auto ck) -> int {
                using S = typename ComponentType<decltype(sk)::value>::T;
                using D = typename ComponentType<decltype(dk)::value>::T;
                using C = typename ComponentType<decltype(ck)::value>::T;
                color_kernel<S, D, C><<<grid, 256, 0, s>>>(plan, (const S*)src->data, src->stride, (D*)dst->data, dst->stride, (int)rows,
                                                            (int)cols);
                ZB_LAUNCHED();
                return ZB_OK;
            });
        });
    });
    if (rc) return rc;
    t_last_kernel = "convert_color";
    return ZB_OK;
}
