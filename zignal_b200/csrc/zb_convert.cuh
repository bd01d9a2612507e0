// zb_convert.cuh -- convertColor(TargetType, pixel) (reference color.zig:108-151) between the five pixel formats, for one pixel on the
// device: the rules of Image.convert (zb_convert.cu), also used by the mixed-type Image.insert (zb_insert_mixed.cu, image.zig:67-95), the
// JPEG codec and quantization.  It is the colour-format conversion of zb_color.cuh with the plan fixed at compile time.
#pragma once
#include "zb_color.cuh"
#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {

// (space, component) of each pixel format
template <int F> struct PixColor;
template <> struct PixColor<ZB_PIX_U8> { static constexpr int space = color::SCALAR, component = color::CU8; };
template <> struct PixColor<ZB_PIX_F32> { static constexpr int space = color::SCALAR, component = color::CF32; };
template <> struct PixColor<ZB_PIX_RGB8> { static constexpr int space = color::RGB, component = color::CU8; };
template <> struct PixColor<ZB_PIX_RGBA8> { static constexpr int space = color::RGBA, component = color::CU8; };
template <> struct PixColor<ZB_PIX_RGBAF32> { static constexpr int space = color::RGBA, component = color::CF32; };

// s: S::N components of the source format, d: D::N components of the destination format (SF != DF)
template <int SF, int DF>
__device__ __forceinline__ void convert_color(const typename Fmt<SF>::CT* s, typename Fmt<DF>::CT* d) {
    using S = PixColor<SF>;
    using D = PixColor<DF>;
    using C = typename color::ComponentType<color::make_plan(S::space, S::component, D::space, D::component).compute>::T;
    color::convert_pixel_static<typename Fmt<SF>::CT, typename Fmt<DF>::CT, C, S::space, S::component, D::space, D::component>(s, d);
}

}  // namespace zb
