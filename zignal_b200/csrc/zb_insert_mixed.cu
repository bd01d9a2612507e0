// zb_insert_mixed.cu -- Image.insert(source: anytype, ...) when the source's pixel type differs from the destination's
// (reference transforms.zig:293-376 with image.zig:67-95 assignPixel): every destination pixel inside the rotated rectangle takes a
// sample of the SOURCE type (interpolate(SourcePixelType, source, x, y, method, .mirror)), which is then
//   * composited when the source is Rgba(u8) and a blend mode is given:  dest = convertColor(DestType, blend(convertColor(Rgba, dest), sample))
//   * converted otherwise:                                               dest = convertColor(DestType, sample).
// Same geometry, same sampler and the same conversion rules as the same-type insert (zb_warp.cu) and Image.convert (zb_convert.cu);
// one kernel templated on (source format, destination format, interpolation method).
#include "zb_warp.h"
#include "zb_sample.cuh"
#include "zb_convert.cuh"
#include "zb_blend.cuh"

namespace zb {
namespace {

__device__ __forceinline__ int mix_patch_col(unsigned t) { return (int)(((t >> 5) & 3u) * 8u + (t & 7u)); }
__device__ __forceinline__ int mix_patch_row(unsigned t) { return (int)((t >> 7) * 4u + ((t >> 3) & 3u)); }

template <int SF, int DF, int METHOD>
__global__ void __launch_bounds__(256) insert_mixed_kernel(SrcView source, typename Fmt<DF>::CT* __restrict__ self, size_t self_stride,
                                                           InsertParams p, const float* __restrict__ lut) {
    using S = Fmt<SF>;
    using D = Fmt<DF>;
    using SCT = typename S::CT;
    using DCT = typename D::CT;
    const int wc = blockIdx.x * 32 + mix_patch_col(threadIdx.x);
    const int wr = ZB_GRID_ROW() * 8 + mix_patch_row(threadIdx.x);
    if (wc >= p.n_c || wr >= p.n_r) return;
    const int r = p.min_r + wr, c = p.min_c + wc;   // destination pixel
    Pix<SCT, S::N> val;
    if (p.copy_rect) {
        val = load_px<SCT, S::N>((const SCT*)source.data, (size_t)(r - p.dst_top) * source.stride + (size_t)(c - p.dst_left));
    } else {
        const float dy = (float)r - p.cy, dx = (float)c - p.cx;
        const float rect_x = p.cos_a * dx + p.sin_a * dy;        // inverse rotation into rectangle space
        const float rect_y = -p.sin_a * dx + p.cos_a * dy;
        if (fabsf(rect_x) > p.half_w || fabsf(rect_y) > p.half_h) return;
        const float norm_x = (rect_x + p.half_w) * p.inv_w;
        const float norm_y = (rect_y + p.half_h) * p.inv_h;
        const float src_x = p.src_cols == 1 ? 0.0f : norm_x * p.fcols1;
        const float src_y = p.src_rows == 1 ? 0.0f : norm_y * p.frows1;
        if (!interpolate<SCT, S::N, METHOD, ZB_BORDER_MIRROR>(source, src_x, src_y, p.mb, p.mc, ZB_BORDER_MIRROR, lut, val)) return;
    }
    DCT* dp = self + ((size_t)r * self_stride + c) * D::N;
    DCT d[D::N];
    if (SF == ZB_PIX_RGBA8 && p.blend != ZB_BLEND_NONE) {   // image.zig:76-87: through Rgba(u8) and back
        if constexpr (SF == ZB_PIX_RGBA8) {
            DCT cur[D::N];
#pragma unroll
            for (int k = 0; k < D::N; ++k) cur[k] = dp[k];
            uint8_t base[4];
            convert_color<DF, ZB_PIX_RGBA8>(cur, base);
            const uint32_t b32 = (uint32_t)base[0] | ((uint32_t)base[1] << 8) | ((uint32_t)base[2] << 16) | ((uint32_t)base[3] << 24);
            const uint32_t o32 = blend_rgba8(b32, val.u, p.blend);
            const uint8_t blended[4] = {(uint8_t)o32, (uint8_t)(o32 >> 8), (uint8_t)(o32 >> 16), (uint8_t)(o32 >> 24)};
            convert_color<ZB_PIX_RGBA8, DF>(blended, d);
        }
    } else {
        convert_color<SF, DF>(val.v, d);                     // :89-93
    }
#pragma unroll
    for (int k = 0; k < D::N; ++k) dp[k] = d[k];
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_insert_from(zb_image* self, int self_pixfmt, const zb_image* source, int source_pixfmt, float rect_l, float rect_t, float rect_r,
                              float rect_b, float angle, float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, int blend_mode,
                              zb_stream stream) {
    if (self_pixfmt == source_pixfmt)
        return zb_insert_blend(self, source, self_pixfmt, rect_l, rect_t, rect_r, rect_b, angle, cos_a, sin_a, method, mitchell_b, mitchell_c, blend_mode,
                               stream);
    if (!self || !source) return ZB_ERR_INVALID_ARGUMENT;
    if (blend_mode < ZB_BLEND_NONE || blend_mode > ZB_BLEND_EXCLUSION) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmtAll, self_pixfmt) || !pixfmt_in(kFmtAll, source_pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (exceeds_int_index(self, self_pixfmt) || exceeds_int_index(source, source_pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (method < ZB_INTERP_NEAREST || method > ZB_INTERP_LANCZOS) return ZB_ERR_INVALID_ARGUMENT;
    if (source->rows == 0 || source->cols == 0) return ZB_OK;   // transforms.zig:294
    if (self->rows == 0 || self->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    InsertParams p;
    if (!insert_plan(self, source, rect_l, rect_t, rect_r, rect_b, angle, cos_a, sin_a, method, mitchell_b, mitchell_c, blend_mode, p)) return ZB_OK;
    const float* lut = nullptr;
    if (method == ZB_INTERP_LANCZOS && (rc = lanczos_lut_device(&lut, s))) return rc;
    t_last_kernel = "insert_mixed";
    SrcView v{source->data, (int)source->rows, (int)source->cols, source->stride};
    const dim3 grid = row_grid(div_up(p.n_c, 32), div_up(p.n_r, 8));
    return dispatch_pixfmt<kFmtAll>(source_pixfmt, [&](auto sf) -> int {
        return dispatch_pixfmt<kFmtAll>(self_pixfmt, [&](auto df) -> int {
            constexpr int SF = decltype(sf)::value, DF = decltype(df)::value;
            if constexpr (SF != DF) {
                return dispatch_method(p.method, [&](auto m) -> int {
                    insert_mixed_kernel<SF, DF, decltype(m)::value><<<grid, 256, 0, s>>>(v, (typename Fmt<DF>::CT*)self->data, (size_t)self->stride,
                                                                                         p, lut);
                    ZB_LAUNCHED();
                    return ZB_OK;
                });
            }
            return ZB_ERR_UNSUPPORTED;
        });
    });
}
