// zb_convert.cu -- Image.convert / convertInto (SURVEY 8(f).4: the pixel-format stage either side of the path; reference
// image.zig:396-421): out[r, c] = convertColor(TargetType, self[r, c]) (color.zig:108-151) between u8, f32, Rgb(u8), Rgba(u8) and
// Rgba(f32).  One elementwise kernel, templated on the (source, destination) pair; the component rules are
//   u8 -> float component   v / 255                      (Gray / Rgb / Rgba .as(f32), color.zig:369-373, 488-493, 550)
//   float -> u8 component   round(255 * clamp(v, 0, 1))  in f32 (.as(u8), :376-379, 496-501, 553); the scalar f32 -> u8 conversion alone
//                           goes through f64 (:114-118)
//   colour -> gray          Rgb(u8): the 16.16 fixed-point BT.709 luma (:1031-1041); float: clamp(lr r + lg g + lb b, 0, 1) (:1043-1045);
//                           Rgba drops its alpha first (:477-479)
//   gray -> colour          replicate, alpha 255 / 1.0 (:1049-1051, :355)
// with every float product and sum separately rounded, so the result is bit-identical to the reference's.
#include "zb_convert.cuh"

namespace zb {
namespace {

template <int SF, int DF>
__global__ void __launch_bounds__(256) convert_kernel(const void* __restrict__ src, size_t src_stride, void* __restrict__ dst, size_t dst_stride,
                                                      int rows, int cols) {
    using S = Fmt<SF>;
    using D = Fmt<DF>;
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = ZB_GRID_ROW();
    if (c >= cols || r >= rows) return;
    const typename S::CT* sp = (const typename S::CT*)src + ((size_t)r * src_stride + c) * S::N;
    typename D::CT* dp = (typename D::CT*)dst + ((size_t)r * dst_stride + c) * D::N;
    typename S::CT s[S::N];
#pragma unroll
    for (int k = 0; k < S::N; ++k) s[k] = sp[k];
    typename D::CT d[D::N];
    convert_color<SF, DF>(s, d);
#pragma unroll
    for (int k = 0; k < D::N; ++k) dp[k] = d[k];
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_convert(const zb_image* src, int src_pixfmt, zb_image* dst, int dst_pixfmt, zb_stream stream) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmtAll, src_pixfmt) || !pixfmt_in(kFmtAll, dst_pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;      // image.zig:397
    if (src_pixfmt == dst_pixfmt) return zb_copy(src, dst, src_pixfmt, stream);                  // :398-399
    if (exceeds_int_index(src, src_pixfmt) || exceeds_int_index(dst, dst_pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    rc = dispatch_pixfmt<kFmtAll>(src_pixfmt, [&](auto sf) -> int {
        return dispatch_pixfmt<kFmtAll>(dst_pixfmt, [&](auto df) -> int {
            constexpr int SF = decltype(sf)::value, DF = decltype(df)::value;
            if constexpr (SF != DF) {
                const dim3 grid = row_grid(div_up(src->cols, 256), src->rows);
                convert_kernel<SF, DF><<<grid, 256, 0, s>>>(src->data, src->stride, dst->data, dst->stride, (int)src->rows, (int)src->cols);
                ZB_LAUNCHED();
                return ZB_OK;
            }
            return ZB_ERR_UNSUPPORTED;
        });
    });
    if (rc) return rc;
    t_last_kernel = "convert";
    return ZB_OK;
}
