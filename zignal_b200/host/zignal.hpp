// zignal.hpp -- C++ host-side mirror of zignal's Image(T) hot methods over the C ABI (header only).
// The reference's toolchain (Zig nightly) is absent from this image, so the host layer above the C ABI
// is provided in C++ (this file) next to the uncompiled Zig shim (zig/zignal_b200.zig).  Method names,
// argument meaning and error behaviour follow reference src/image.zig:523-1147.  Image<T> wraps HOST buffers (each call is the literal
// drop-in: upload, kernel, download); DeviceImage<T> wraps device buffers for resident chains.  tests/test_host_cpp_mirror.py compiles this
// header with -Wall -Wextra -Werror for every pixel type and links it against the library.
#pragma once
#include <cmath>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/zignal_b200.h"

namespace zignal {

struct Rgb8 { uint8_t r, g, b; };
struct Rgba8 { uint8_t r, g, b, a; };
struct RgbaF32 { float r, g, b, a; };

template <typename T> constexpr int pixfmt_of();
template <> constexpr int pixfmt_of<uint8_t>() { return ZB_PIX_U8; }
template <> constexpr int pixfmt_of<float>() { return ZB_PIX_F32; }
template <> constexpr int pixfmt_of<Rgb8>() { return ZB_PIX_RGB8; }
template <> constexpr int pixfmt_of<Rgba8>() { return ZB_PIX_RGBA8; }
template <> constexpr int pixfmt_of<RgbaF32>() { return ZB_PIX_RGBAF32; }

// The colour types of color.zig, each with its ColorSpace tag and its fields in declaration order (Rgba is packed r, g, b, a).
// Component types: uint8_t, float, double; the reference allows uint8_t only for Gray, Rgb, Rgba and Ycbcr.
#define ZIGNAL_COLOR3(Name, SPACE, A, B, C)                                                    \
    template <typename T> struct Name { static constexpr int space = SPACE; using component = T; T A, B, C; };
template <typename T> struct Gray { static constexpr int space = ZB_SPACE_GRAY; using component = T; T y; };
template <typename T> struct Rgba { static constexpr int space = ZB_SPACE_RGBA; using component = T; T r, g, b, a; };
ZIGNAL_COLOR3(Rgb, ZB_SPACE_RGB, r, g, b)
ZIGNAL_COLOR3(Hsl, ZB_SPACE_HSL, h, s, l)
ZIGNAL_COLOR3(Hsv, ZB_SPACE_HSV, h, s, v)
ZIGNAL_COLOR3(Xyz, ZB_SPACE_XYZ, x, y, z)
ZIGNAL_COLOR3(Lab, ZB_SPACE_LAB, l, a, b)
ZIGNAL_COLOR3(Lch, ZB_SPACE_LCH, l, c, h)
ZIGNAL_COLOR3(Lms, ZB_SPACE_LMS, l, m, s)
ZIGNAL_COLOR3(Oklab, ZB_SPACE_OKLAB, l, a, b)
ZIGNAL_COLOR3(Oklch, ZB_SPACE_OKLCH, l, c, h)
ZIGNAL_COLOR3(Xyb, ZB_SPACE_XYB, x, y, b)
ZIGNAL_COLOR3(Ycbcr, ZB_SPACE_YCBCR, y, cb, cr)
#undef ZIGNAL_COLOR3

template <typename C> constexpr int component_of() {
    static_assert(std::is_same<C, uint8_t>::value || std::is_same<C, float>::value || std::is_same<C, double>::value, "component type");
    return std::is_same<C, uint8_t>::value ? ZB_COMPONENT_U8 : std::is_same<C, float>::value ? ZB_COMPONENT_F32 : ZB_COMPONENT_F64;
}
struct ColorFormat { int space, component; };
// (space, component) of a pixel type, as zb_color_image carries it.
template <typename T> constexpr ColorFormat color_format_of() {
    if constexpr (std::is_arithmetic<T>::value) return {ZB_SPACE_SCALAR, component_of<T>()};
    else if constexpr (std::is_same<T, Rgb8>::value) return {ZB_SPACE_RGB, ZB_COMPONENT_U8};
    else if constexpr (std::is_same<T, Rgba8>::value) return {ZB_SPACE_RGBA, ZB_COMPONENT_U8};
    else if constexpr (std::is_same<T, RgbaF32>::value) return {ZB_SPACE_RGBA, ZB_COMPONENT_F32};
    else return {T::space, component_of<typename T::component>()};
}
// The five pixel types every image entry point takes.
template <typename T> constexpr bool has_pixfmt() {
    return std::is_same<T, uint8_t>::value || std::is_same<T, float>::value || std::is_same<T, Rgb8>::value ||
           std::is_same<T, Rgba8>::value || std::is_same<T, RgbaF32>::value;
}

struct Error : std::runtime_error {
    int status;
    explicit Error(int s) : std::runtime_error(std::string("zignal error.") + zb_status_name(s)), status(s) {}
};
inline void check(int status) { if (status != ZB_OK) throw Error(status); }

enum class BorderMode { zero = 0, replicate = 1, mirror = 2, wrap = 3 };
struct Interpolation {
    int tag = ZB_INTERP_BILINEAR;
    float b = 1.0f / 3.0f, c = 1.0f / 3.0f;
    static Interpolation nearest() { return {ZB_INTERP_NEAREST}; }
    static Interpolation bilinear() { return {ZB_INTERP_BILINEAR}; }
    static Interpolation bicubic() { return {ZB_INTERP_BICUBIC}; }
    static Interpolation catmull_rom() { return {ZB_INTERP_CATMULL_ROM}; }
    static Interpolation mitchell(float b, float c) { return {ZB_INTERP_MITCHELL, b, c}; }
    static Interpolation lanczos() { return {ZB_INTERP_LANCZOS}; }
};

// Image<T> over HOST memory: every method is the literal drop-in (H2D + kernel + D2H inside the call).
template <typename T>
struct Image {
    uint32_t rows = 0, cols = 0;
    T* data = nullptr;
    size_t stride = 0;  // pixels

    zb_image raw() const { return zb_image{(void*)data, rows, cols, (uint64_t)stride}; }
    bool hasSameShape(const Image& o) const { return rows == o.rows && cols == o.cols; }

    void gaussianBlur(Image out, float sigma) const { auto a = raw(), d = out.raw(); check(zb_host_gaussian_blur(&a, &d, pixfmt_of<T>(), sigma)); }
    void convolveSeparable(Image out, const std::vector<float>& kx, const std::vector<float>& ky, BorderMode border) const {
        auto a = raw(), d = out.raw();
        check(zb_host_conv_separable(&a, &d, pixfmt_of<T>(), kx.data(), (int)kx.size(), ky.data(), (int)ky.size(), (int)border));
    }
    template <size_t KH, size_t KW>
    void convolve(Image out, const float (&kernel)[KH][KW], BorderMode border) const {
        auto a = raw(), d = out.raw();
        check(zb_host_convolve(&a, &d, pixfmt_of<T>(), &kernel[0][0], (int)KH, (int)KW, (int)border));
    }
    void boxBlur(Image out, uint32_t radius) const { auto a = raw(), d = out.raw(); check(zb_host_box_blur(&a, &d, pixfmt_of<T>(), radius)); }
    void sharpen(Image out, size_t radius) const { auto a = raw(), d = out.raw(); check(zb_host_sharpen(&a, &d, pixfmt_of<T>(), (uint32_t)radius)); }
    void resize(Image out, Interpolation m) const { auto a = raw(), d = out.raw(); zb_host_resize(&a, &d, pixfmt_of<T>(), m.tag, m.b, m.c); }
    void rotateInto(Image out, float angle, Interpolation m, BorderMode border) const {
        auto a = raw(), d = out.raw();
        zb_host_rotate_into(&a, &d, pixfmt_of<T>(), angle, m.tag, m.b, m.c, (int)border);
    }
    struct Bounds { uint32_t rows, cols; };
    Bounds rotateBounds(float angle) const { Bounds b{}; zb_rotate_bounds(rows, cols, angle, &b.rows, &b.cols); return b; }
    // transform: {m00,m01,m10,m11,b0,b1} (similarity/affine) or 9 values (projective)
    void warp(Image out, int xform_kind, const float* m, Interpolation method) const {
        auto a = raw(), d = out.raw();
        zb_host_warp(&a, &d, pixfmt_of<T>(), xform_kind, m, method.tag, method.b, method.c);
    }
};

enum class Blending { none = 0, normal, multiply, screen, overlay, soft_light, hard_light, color_dodge, color_burn, darken, lighten, difference, exclusion };
struct Rect { float l, t, r, b; };   // geometry/Rectangle.zig (f32; r and b exclusive)

// BinaryKernel (binary.zig:9-33): odd x odd structuring element, non-zero = on; the constructor checks what Kernel.init checks.
struct BinaryKernel {
    uint32_t rows = 0, cols = 0;
    std::vector<uint8_t> data;
    BinaryKernel(uint32_t r, uint32_t c, std::vector<uint8_t> d) : rows(r), cols(c), data(std::move(d)) {
        if (r == 0 || c == 0 || r % 2 == 0 || c % 2 == 0 || data.size() != (size_t)r * c) throw Error(ZB_ERR_INVALID_KERNEL_SIZE);
    }
};

// ShenCastan (ShenCastan.zig:9-37): options of shenCastan with the reference's defaults, and its presets (:51-99).
struct ShenCastan {
    float smooth = 0.9f;        // ISEF smoothing factor, 0 < smooth < 1
    size_t window_size = 7;     // odd, >= 3
    float high_ratio = 0.99f;   // percentile of the high threshold, 0 < high_ratio < 1
    float low_rel = 0.5f;       // low threshold = low_rel * high threshold, 0 < low_rel < 1
    bool hysteresis = true;
    bool use_nms = false;
    static ShenCastan defaults() { return {}; }
    static ShenCastan low_noise() { ShenCastan o; o.smooth = 0.95f; o.high_ratio = 0.98f; return o; }
    static ShenCastan high_noise() { ShenCastan o; o.smooth = 0.7f; o.window_size = 11; return o; }
    static ShenCastan heavy_smooth() { ShenCastan o; o.smooth = 0.5f; o.window_size = 9; o.high_ratio = 0.95f; return o; }
    static ShenCastan sensitive() { ShenCastan o; o.high_ratio = 0.97f; o.low_rel = 0.4f; return o; }
    static ShenCastan thin() { ShenCastan o; o.use_nms = true; return o; }
    static ShenCastan strong_only() { ShenCastan o; o.hysteresis = false; return o; }
};

// FloodFillOptions (image/flood_fill.zig:5-26): the reference's defaults.
struct FloodFillOptions {
    enum class Connectivity : int { four = 4, eight = 8 };
    enum class ThresholdMode : int { seed = ZB_FLOOD_SEED, neighbor = ZB_FLOOD_NEIGHBOR };
    double threshold = 0;                          // maximum colour distance for a neighbour to be filled
    Connectivity connectivity = Connectivity::four;
    ThresholdMode mode = ThresholdMode::seed;      // compare candidates with the seed, or with the neighbour they spread from
};

// DeviceImage<T>: the same {rows, cols, data, stride} struct over DEVICE memory, for callers that keep a chain of operations resident
// (SURVEY 8(f)).  Non-owning, like the reference's views; every method enqueues on `stream` and mirrors the Zig method it is named after
// (image.zig line in the comment).  Methods returning a double wait for the stream.
template <typename T>
struct DeviceImage {
    uint32_t rows = 0, cols = 0;
    T* data = nullptr;     // device pointer (zb_malloc / cudaMalloc)
    size_t stride = 0;     // pixels
    zb_stream stream = nullptr;

    zb_image raw() const { return zb_image{(void*)data, rows, cols, (uint64_t)stride}; }
    DeviceImage view(uint32_t l, uint32_t t, uint32_t r, uint32_t b) const {                       // :426-430
        return DeviceImage{b - t, r - l, data + (size_t)t * stride + l, stride, stream};
    }
    void copy(DeviceImage out) const { auto a = raw(), d = out.raw(); check(zb_copy(&a, &d, pixfmt_of<T>(), stream)); }              // :375
    zb_color_image color_raw() const {
        constexpr ColorFormat f = color_format_of<T>();
        return zb_color_image{(void*)data, rows, cols, (uint64_t)stride, f.space, f.component};
    }
    // :396.  Between two of the five pixel types this is zb_convert; any other pair of colour types goes through zb_convert_color.
    template <typename U>
    void convertInto(DeviceImage<U> out) const {
        if constexpr (has_pixfmt<T>() && has_pixfmt<U>()) {
            auto a = raw(), d = out.raw();
            check(zb_convert(&a, pixfmt_of<T>(), &d, pixfmt_of<U>(), stream));
        } else {
            auto a = color_raw(), d = out.color_raw();
            check(zb_convert_color(&a, &d, stream));
        }
    }
    void gaussianBlur(DeviceImage out, float sigma) const { auto a = raw(), d = out.raw(); check(zb_gaussian_blur(&a, &d, pixfmt_of<T>(), sigma, stream)); }   // :954
    void convolveSeparable(DeviceImage out, const std::vector<float>& kx, const std::vector<float>& ky, BorderMode border) const {     // :935
        auto a = raw(), d = out.raw();
        check(zb_conv_separable(&a, &d, pixfmt_of<T>(), kx.data(), (int)kx.size(), ky.data(), (int)ky.size(), (int)border, stream));
    }
    template <size_t KH, size_t KW>
    void convolve(DeviceImage out, const float (&kernel)[KH][KW], BorderMode border) const {                                          // :917
        auto a = raw(), d = out.raw();
        check(zb_convolve(&a, &d, pixfmt_of<T>(), &kernel[0][0], (int)KH, (int)KW, (int)border, stream));
    }
    void boxBlur(DeviceImage out, uint32_t radius) const { auto a = raw(), d = out.raw(); check(zb_box_blur(&a, &d, pixfmt_of<T>(), radius, stream)); }      // :635
    void sharpen(DeviceImage out, uint32_t radius) const { auto a = raw(), d = out.raw(); check(zb_sharpen(&a, &d, pixfmt_of<T>(), radius, stream)); }       // :785
    void medianBlur(DeviceImage out, uint32_t radius) const { order(out, radius, ZB_ORDER_PERCENTILE, 0.5, BorderMode::mirror); }                             // :650
    void percentileBlur(DeviceImage out, uint32_t radius, double percentile, BorderMode border) const { order(out, radius, ZB_ORDER_PERCENTILE, percentile, border); }   // :672
    void minBlur(DeviceImage out, uint32_t radius, BorderMode border) const { order(out, radius, ZB_ORDER_PERCENTILE, 0.0, border); }                         // :696
    void maxBlur(DeviceImage out, uint32_t radius, BorderMode border) const { order(out, radius, ZB_ORDER_PERCENTILE, 1.0, border); }                         // :719
    void midpointBlur(DeviceImage out, uint32_t radius, BorderMode border) const { order(out, radius, ZB_ORDER_MIDPOINT, 0.0, border); }                      // :742
    void alphaTrimmedMeanBlur(DeviceImage out, uint32_t radius, double trim, BorderMode border) const { order(out, radius, ZB_ORDER_ALPHA_TRIMMED, trim, border); }   // :767
    void motionBlurLinear(DeviceImage out, float angle, uint32_t distance) const {                                                                           // motion_blur.zig:65
        auto a = raw(), d = out.raw();
        check(zb_motion_blur_linear(&a, &d, pixfmt_of<T>(), angle, std::cos(angle), std::sin(angle), distance, stream));
    }
    void motionBlurRadial(DeviceImage out, float center_x, float center_y, float strength, bool spin) const {                                                // motion_blur.zig:252
        auto a = raw(), d = out.raw();
        check(zb_motion_blur_radial(&a, &d, pixfmt_of<T>(), center_x, center_y, strength, spin ? 1 : 0, stream));
    }
    void resize(DeviceImage out, Interpolation m) const { auto a = raw(), d = out.raw(); check(zb_resize(&a, &d, pixfmt_of<T>(), m.tag, m.b, m.c, stream)); }   // :523
    void rotateInto(DeviceImage out, float angle, Interpolation m, BorderMode border) const {                                                               // :564
        auto a = raw(), d = out.raw();
        check(zb_rotate_into(&a, &d, pixfmt_of<T>(), angle, m.tag, m.b, m.c, (int)border, stream));
    }
    void warp(DeviceImage out, int xform_kind, const float* m, Interpolation method) const {                                                                // :621
        auto a = raw(), d = out.raw();
        check(zb_warp(&a, &d, pixfmt_of<T>(), xform_kind, m, method.tag, method.b, method.c, stream));
    }
    void extract(DeviceImage out, Rect rect, float angle, Interpolation m, BorderMode border) const {                                                       // :594
        auto a = raw(), d = out.raw();
        check(zb_extract(&a, &d, pixfmt_of<T>(), rect.l, rect.t, rect.r, rect.b, angle, std::cos(angle), std::sin(angle), m.tag, m.b, m.c, (int)border, stream));
    }
    void insert(DeviceImage source, Rect rect, float angle, Interpolation m, Blending blend) {                                                              // :604
        auto d = raw(), a = source.raw();
        check(zb_insert_blend(&d, &a, pixfmt_of<T>(), rect.l, rect.t, rect.r, rect.b, angle, std::cos(angle), std::sin(angle), m.tag, m.b, m.c, (int)blend, stream));
    }
    void sobel(DeviceImage<uint8_t> out) const { auto a = raw(), d = out.raw(); check(zb_sobel(&a, &d, pixfmt_of<T>(), stream)); }                            // :999
    void canny(DeviceImage<uint8_t> out, float sigma, float low, float high) const {                                                                        // :1041
        auto a = raw(), d = out.raw();
        check(zb_canny(&a, &d, pixfmt_of<T>(), sigma, low, high, stream));
    }
    void shenCastan(DeviceImage<uint8_t> out, const ShenCastan& opts) const {                                                                         // :1015
        auto a = raw(), d = out.raw();
        check(zb_shen_castan(&a, &d, pixfmt_of<T>(), opts.smooth, (uint64_t)opts.window_size, opts.high_ratio, opts.low_rel, opts.hysteresis ? 1 : 0,
                             opts.use_nms ? 1 : 0, stream));
    }
    double psnr(DeviceImage other) const { return metric(zb_psnr, other); }                                                                                  // :1105
    double ssim(DeviceImage other) const { return metric(zb_ssim, other); }                                                                                  // :1126
    double meanPixelError(DeviceImage other) const { return metric(zb_mean_pixel_error, other); }                                                            // :1145
    // 8-bit histogram family (u8, Rgb8, Rgba8) and Image(u8) binary operations (image.zig:804-914, 1161-1185)
    std::vector<uint32_t> histogram() const {                                           // :1161, channels x 256 counts; waits for the stream
        std::vector<uint32_t> counts(256 * (size_t)(pixfmt_of<T>() == ZB_PIX_U8 ? 1 : pixfmt_of<T>() == ZB_PIX_RGB8 ? 3 : 4));
        auto a = raw();
        check(zb_histogram(&a, pixfmt_of<T>(), counts.data(), stream));
        return counts;
    }
    void autocontrast(float cutoff) const { auto a = raw(); check(zb_autocontrast(&a, pixfmt_of<T>(), cutoff, stream)); }                                 // :804
    void equalize() const { auto a = raw(); check(zb_equalize(&a, pixfmt_of<T>(), stream)); }                                                             // :824
    // :1139, diff.zig:27-203: out may be *this or other; returns DiffResult's values (waits for the stream).
    zb_diff_stats diff(DeviceImage out, DeviceImage other, float threshold = 0, float scale = 1, bool binary = false, bool force_opaque = false) const {
        auto a = raw(), b = other.raw(), o = out.raw();
        zb_diff_stats st{};
        check(zb_diff(&a, &b, &o, pixfmt_of<T>(), threshold, scale, binary ? 1 : 0, force_opaque ? 1 : 0, &st, stream));
        return st;
    }
    // jpeg.encode (codecs/jpeg.zig:307-325): the baseline JPEG file of this device image, byte-identical to zignal's encoder (waits
    // for the stream).  The first call's capacity is the raw pixel size plus the header; a larger stream is fetched once more.
    std::vector<uint8_t> encode_jpeg(uint8_t quality = 90, zb_jpeg_subsampling subsampling = ZB_JPEG_YUV420, uint16_t density_dpi = 72,
                                     const std::string* comment = nullptr) const {
        auto a = raw();
        zb_jpeg_options o{quality, (uint8_t)subsampling, density_dpi, comment ? (const uint8_t*)comment->data() : nullptr,
                          comment ? (uint32_t)comment->size() : 0u};
        std::vector<uint8_t> out((size_t)rows * cols * sizeof(T) + 1024 + (comment ? comment->size() : 0));
        uint64_t len = 0;
        int rc = zb_jpeg_encode(&a, pixfmt_of<T>(), &o, out.data(), out.size(), &len, stream);
        if (rc == ZB_ERR_OUT_OF_MEMORY && len > out.size()) {
            out.resize(len);
            rc = zb_jpeg_encode(&a, pixfmt_of<T>(), &o, out.data(), out.size(), &len, stream);
        }
        check(rc);
        out.resize(len);
        return out;
    }
    // jpeg.loadFromBytes (codecs/jpeg.zig:2825-2851) into this device image, which must have the file's rows and cols (zb_jpeg_info
    // gives them); entropy decoding runs on the device.  limits: NULL for jpeg.DecodeLimits' defaults.  Waits for the stream.
    void decode_jpeg(const uint8_t* data, size_t len, const zb_jpeg_limits* limits = nullptr) const {
        auto a = raw();
        check(zb_jpeg_decode(data, len, limits, &a, pixfmt_of<T>(), stream));
    }
    // :1190-1247 into an Rgb(u8) image of the same shape; lut768 from zb_colormap_lut (jet / heat / turbo) or the caller's table.
    // A NaN bound is a bound; pass has_min / has_max = false for the image's own minimum / maximum.
    void applyColormap(DeviceImage<Rgb8> out, const uint8_t* lut768, bool has_min = false, double min = 0, bool has_max = false,
                       double max = 0) const {
        auto a = raw(), d = out.raw();
        check(zb_apply_colormap(&a, pixfmt_of<T>(), lut768, has_min ? 1 : 0, min, has_max ? 1 : 0, max, &d, stream));
    }
    void flipLeftRight() const { auto a = raw(); check(zb_flip_left_right(&a, pixfmt_of<T>(), stream)); }                                  // :480
    void flipTopBottom() const { auto a = raw(); check(zb_flip_top_bottom(&a, pixfmt_of<T>(), stream)); }                                  // :485
    void invert() const {                                                                                                                  // :494
        static_assert(!std::is_same<T, float>::value, "invert() requires pixel types with an invert() method or u8 grayscale pixels");
        auto a = raw();
        check(zb_invert(&a, pixfmt_of<T>(), stream));
    }
    // :831-840, flood_fill.zig:59-131: in place; FloodFillOptions below.  OutOfBounds (a seed outside the image) throws Error.
    void floodFill(uint32_t start_row, uint32_t start_col, T fill_value, FloodFillOptions options = {}) const {
        auto a = raw();
        check(zb_flood_fill(&a, pixfmt_of<T>(), start_row, start_col, &fill_value, options.threshold, (int)options.connectivity,
                            (int)options.mode, stream));
    }
    // quantize.zig:175-412 medianCut: fills the host `palette` (cap x 3 bytes) and returns the count.  Waits for the stream.
    uint32_t medianCut(uint8_t* palette, uint32_t cap, uint16_t max_colors) const {
        auto a = raw();
        uint32_t n = 0;
        check(zb_median_cut(&a, pixfmt_of<T>(), max_colors, palette, cap, &n, stream));
        return n;
    }
    // dither.zig:34-41 dither.apply in place on an Rgb(u8) image; `lut` is a device table from zb_color_lut.
    void dither(const uint8_t* palette, uint32_t n, const uint8_t* lut, int mode) const {
        auto a = raw();
        check(zb_dither(&a, pixfmt_of<T>(), palette, n, lut, mode, stream));
    }
    // quantize.zig:163-168 ColorLookupTable.lookup(convertColor(Rgb, px)) per pixel into a u8 index image of the same shape.
    void paletteIndices(const uint8_t* lut, DeviceImage<uint8_t> out) const {
        auto a = raw(), d = out.raw();
        check(zb_palette_lookup(&a, pixfmt_of<T>(), lut, &d, stream));
    }
    uint8_t thresholdOtsu(DeviceImage out) const {                                                                                                        // :845
        static_assert(std::is_same<T, uint8_t>::value, "thresholdOtsu is only available for Image(u8)");
        auto a = raw(), d = out.raw();
        uint8_t t = 0;
        check(zb_threshold_otsu(&a, &d, &t, stream));
        return t;
    }
    void thresholdAdaptiveMean(DeviceImage out, uint32_t radius, float c) const {                                                                         // :858
        static_assert(std::is_same<T, uint8_t>::value, "thresholdAdaptiveMean is only available for Image(u8)");
        auto a = raw(), d = out.raw();
        check(zb_threshold_adaptive_mean(&a, &d, radius, c, stream));
    }
    void dilateBinary(DeviceImage out, const BinaryKernel& k, uint32_t iterations) const { morph(out, k, iterations, ZB_MORPH_DILATE); }                 // :870
    void erodeBinary(DeviceImage out, const BinaryKernel& k, uint32_t iterations) const { morph(out, k, iterations, ZB_MORPH_ERODE); }                   // :881
    void openBinary(DeviceImage out, const BinaryKernel& k, uint32_t iterations) const { morph(out, k, iterations, ZB_MORPH_OPEN); }                     // :892
    void closeBinary(DeviceImage out, const BinaryKernel& k, uint32_t iterations) const { morph(out, k, iterations, ZB_MORPH_CLOSE); }                   // :903

private:
    void morph(DeviceImage out, const BinaryKernel& k, uint32_t iterations, int op) const {
        static_assert(std::is_same<T, uint8_t>::value, "binary morphology is only available for Image(u8)");
        auto a = raw(), d = out.raw();
        check(zb_morph_binary(&a, &d, k.data.data(), k.rows, k.cols, iterations, op, stream));
    }
    void order(DeviceImage out, uint32_t radius, int mode, double param, BorderMode border) const {
        auto a = raw(), d = out.raw();
        check(zb_order_blur(&a, &d, pixfmt_of<T>(), radius, mode, param, (int)border, stream));
    }
    template <typename F>
    double metric(F fn, DeviceImage other) const {
        auto a = raw(), b = other.raw();
        double out = 0.0;
        check(fn(&a, &b, pixfmt_of<T>(), &out, stream));
        return out;
    }
};

// HoughTransform (image/hough.zig:10-257) over device images.  The accumulator is a size x size DeviceImage<uint32_t> (a plain
// {rows, cols, data, stride, stream} holder; only its fields are used) that compute ADDS to, as in the reference: zero it first.
// findLines waits for the accumulator's stream.
class HoughTransform {
public:
    using Line = zb_hough_line;   // Line, :13-25, with the points flattened

    explicit HoughTransform(uint32_t size) { check(zb_hough_create(size, nullptr, nullptr, &h_)); size_ = size; }   // init, :38-66
    ~HoughTransform() { zb_hough_destroy(h_); }                                                                        // deinit, :68-72
    HoughTransform(const HoughTransform&) = delete;
    HoughTransform& operator=(const HoughTransform&) = delete;

    uint32_t size() const { return size_; }
    uint32_t evenSize() const { return size_ - size_ % 2; }

    // :75-139; box (l, t, r, b) with r, b exclusive
    void compute(const DeviceImage<uint8_t>& edges, uint32_t l, uint32_t t, uint32_t r, uint32_t b, DeviceImage<uint32_t> accumulator) const {
        auto e = edges.raw();
        auto a = accumulator.raw();
        check(zb_hough_compute(h_, &e, l, t, r, b, &a, accumulator.stream));
    }
    // :142-204
    std::vector<Line> findLines(DeviceImage<uint32_t> accumulator, uint32_t threshold, float angle_nms_thresh, float radius_nms_thresh) const {
        auto a = accumulator.raw();
        std::vector<Line> lines(1024);
        uint32_t n = 0;
        check(zb_hough_find_lines(h_, &a, threshold, angle_nms_thresh, radius_nms_thresh, lines.data(), (uint32_t)lines.size(), &n, accumulator.stream));
        if (n > lines.size()) {
            lines.resize(n);
            check(zb_hough_find_lines(h_, &a, threshold, angle_nms_thresh, radius_nms_thresh, lines.data(), n, &n, accumulator.stream));
        }
        lines.resize(n);
        return lines;
    }

private:
    zb_hough* h_ = nullptr;
    uint32_t size_ = 0;
};

// A view of host bytes (std::span<const uint8_t> before C++20).
struct Bytes {
    const uint8_t* data = nullptr;
    size_t size = 0;
};
// jpeg.loadFromBytes for many files in one call (zb_jpeg_decode_batch): files[i] into out[i], which must have that file's rows and
// cols.  Returns each file's status (ZB_OK, or what DeviceImage::decode_jpeg would throw for it); throws only for the call's own
// errors.  limits: NULL for jpeg.DecodeLimits' defaults.  Waits for the stream.
template <typename T>
std::vector<int> decode_jpeg_batch(const std::vector<Bytes>& files, const std::vector<DeviceImage<T>>& out,
                                   const zb_jpeg_limits* limits = nullptr, zb_stream stream = nullptr) {
    if (files.size() != out.size()) throw Error(ZB_ERR_INVALID_ARGUMENT);
    std::vector<const uint8_t*> data(files.size());
    std::vector<uint64_t> len(files.size());
    std::vector<zb_image> dst(files.size());
    std::vector<int> fmt(files.size(), pixfmt_of<T>()), status(files.size());
    for (size_t i = 0; i < files.size(); ++i) {
        data[i] = files[i].data;
        len[i] = files[i].size;
        dst[i] = out[i].raw();
    }
    check(zb_jpeg_decode_batch((uint32_t)files.size(), data.data(), len.data(), limits, dst.data(), fmt.data(), status.data(), stream));
    return status;
}

// Matrix.eigh (matrix/eigen.zig:34): row-major n x n symmetric input -> eigenvalues ascending + eigenvectors as columns.
struct Eigh {
    std::vector<double> values, vectors;
};
inline Eigh eigh(const std::vector<double>& a, uint32_t n) {
    Eigh e{std::vector<double>(n), std::vector<double>((size_t)n * n)};
    check(zb_eigh_f64(a.data(), n, n, e.values.data(), e.vectors.data()));
    return e;
}

// Matrix.lu / LuResult.solve / det / inv / chol (Matrix.zig:67-85, 376-441, 511-583, 1156-1365) on DEVICE row-major n x n matrices.
// lu is packed (strict lower triangle: L, unit diagonal implied; upper: U); Matrix.solve is lu followed by luSolve.  Each call returns
// after the stream has finished; the statuses throw (Singular, NotPositiveDefinite, ...).
inline double lu(const double* a, uint32_t n, double* lu_out, uint32_t* perm, zb_stream s = nullptr) {
    double sign = 1; check(zb_lu_f64(a, n, n, lu_out, perm, &sign, s)); return sign;
}
inline float lu(const float* a, uint32_t n, float* lu_out, uint32_t* perm, zb_stream s = nullptr) {
    float sign = 1; check(zb_lu_f32(a, n, n, lu_out, perm, &sign, s)); return sign;
}
inline void luSolve(const double* lu_in, const uint32_t* perm, uint32_t n, const double* b, uint32_t k, double* x, zb_stream s = nullptr) {
    check(zb_lu_solve_f64(lu_in, perm, n, b, n, k, x, s));
}
inline void luSolve(const float* lu_in, const uint32_t* perm, uint32_t n, const float* b, uint32_t k, float* x, zb_stream s = nullptr) {
    check(zb_lu_solve_f32(lu_in, perm, n, b, n, k, x, s));
}
inline double det(const double* a, uint32_t n, zb_stream s = nullptr) { double d = 0; check(zb_det_f64(a, n, n, &d, s)); return d; }
inline float det(const float* a, uint32_t n, zb_stream s = nullptr) { float d = 0; check(zb_det_f32(a, n, n, &d, s)); return d; }
inline void inv(const double* a, uint32_t n, double* out, zb_stream s = nullptr) { check(zb_inv_f64(a, n, n, out, s)); }
inline void inv(const float* a, uint32_t n, float* out, zb_stream s = nullptr) { check(zb_inv_f32(a, n, n, out, s)); }
inline void chol(const double* a, uint32_t n, double* l, zb_stream s = nullptr) { check(zb_chol_f64(a, n, n, l, s)); }
inline void chol(const float* a, uint32_t n, float* l, zb_stream s = nullptr) { check(zb_chol_f32(a, n, n, l, s)); }

}  // namespace zignal
