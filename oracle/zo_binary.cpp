// zo_binary.cpp -- CPU oracle for Image.histogram / autocontrast / equalize / thresholdOtsu / thresholdAdaptiveMean and binary
// morphology.  TEST INFRASTRUCTURE ONLY (see zignal_oracle.h).  Restates image.zig:1161-1185 (histogram), image/histogram.zig:19-162
// (findCutoffMin / findCutoffMax), image/enhancement.zig:11-252 (autocontrast, equalize), image/binary.zig:9-280 (Kernel,
// thresholdOtsu, thresholdAdaptiveMean with Integral.sum, dilate / erode / open / close) and image.zig:845-914.
//
// One stated deviation: equalize forms (cdf[i] - cdf_min) * 255 in 64 bits (enhancement.zig:121,218 is a u32 product, which
// overflows -- a trap or undefined behaviour in Zig -- once total - cdf_min exceeds 16,843,009).
//
// Built on its own into oracle/libzo_binary.so (Makefile; ctypes binding in tests/binary_oracle.py), so the entry points and the
// status codes this family adds are declared here rather than in zignal_oracle.h.
#include <cmath>
#include <vector>

#include "zo_common.h"

extern "C" {
/* Status codes of this family (Zig error names; the same values as zignal_b200.h). */
enum { ZO_ERR_INVALID_CUTOFF = 21 /* enhancement.zig:17 */, ZO_ERR_INVALID_RADIUS = 22 /* binary.zig:93 */,
       ZO_ERR_INVALID_KERNEL_SIZE = 23 /* binary.zig:23-25 */ };
enum { ZO_MORPH_DILATE = 0, ZO_MORPH_ERODE = 1, ZO_MORPH_OPEN = 2, ZO_MORPH_CLOSE = 3 };
int zo_histogram(const zo_image* src, int pixfmt, uint32_t* counts);
int zo_autocontrast(zo_image* img, int pixfmt, float cutoff);
int zo_equalize(zo_image* img, int pixfmt);
int zo_threshold_otsu(const zo_image* src, zo_image* dst, uint8_t* threshold);
int zo_threshold_adaptive_mean(const zo_image* src, zo_image* dst, uint32_t radius, float c);
int zo_morph_binary(const zo_image* src, zo_image* dst, const uint8_t* kernel, uint32_t kernel_rows, uint32_t kernel_cols,
                    uint32_t iterations, int op);
}

namespace zo {

// Integral.compute of an Image(u8) plane (integral.zig:41-78): sequential f32 running sum along each row, then row r-1 added into
// row r.  Once sums pass 2^24 this order is part of the result.
static void integral_plane_u8(const zo_image* src, float* sat) {
    const size_t rows = src->rows, cols = src->cols;
    const uint8_t* base = (const uint8_t*)src->data;
    for (size_t r = 0; r < rows; ++r) {
        float tmp = 0;
        for (size_t c = 0; c < cols; ++c) {
            tmp += (float)base[r * src->stride + c];
            sat[r * cols + c] = tmp;
        }
    }
    for (size_t r = 1; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) sat[r * cols + c] = sat[(r - 1) * cols + c] + sat[r * cols + c];   // :69 prev + curr
}

// image.zig:1161-1185: the pixel iterator visits the view's own pixels, every channel counted (Rgba alpha too).
static void histogram(const zo_image* src, int ch, uint32_t* counts) {
    for (int i = 0; i < ch * 256; ++i) counts[i] = 0;
    const uint8_t* base = (const uint8_t*)src->data;
    for (size_t r = 0; r < src->rows; ++r)
        for (size_t c = 0; c < src->cols; ++c)
            for (int k = 0; k < ch; ++k) counts[k * 256 + base[(r * src->stride + c) * ch + k]] += 1;
}

// histogram.zig:123-142
static uint8_t find_cutoff_min(const uint32_t* values, uint32_t cutoff_pixels) {
    if (cutoff_pixels == 0) {
        for (int i = 0; i < 256; ++i)
            if (values[i] > 0) return (uint8_t)i;
        return 0;
    }
    uint32_t cumulative = 0;
    for (int i = 0; i < 256; ++i) {
        cumulative += values[i];
        if (cumulative > cutoff_pixels) return (uint8_t)i;
    }
    return 255;
}

// histogram.zig:145-162 (`while (i > 0)`: bin 0 is never visited)
static uint8_t find_cutoff_max(const uint32_t* values, uint32_t cutoff_pixels) {
    if (cutoff_pixels == 0) {
        for (size_t i = 255; i > 0; --i)
            if (values[i] > 0) return (uint8_t)i;
        return 0;
    }
    uint32_t cumulative = 0;
    for (size_t i = 255; i > 0; --i) {
        cumulative += values[i];
        if (cumulative > cutoff_pixels) return (uint8_t)i;
    }
    return 0;
}

// enhancement.zig:55-62 remap (the u8 path at :31-39 is the same sequence)
static uint8_t remap(uint8_t val, uint8_t mn, uint8_t mx) {
    const uint8_t clamped = std::max(mn, std::min(mx, val));
    const uint8_t range = mx > mn ? (uint8_t)(mx - mn) : (uint8_t)1;
    const float normalized = (float)(uint8_t)(clamped - mn) / (float)range;
    return (uint8_t)std::round(normalized * 255.0f);   // @round: half away from zero
}

// enhancement.zig:198-216 createLut (u8 path :102-127), with the 64-bit numerator
static void equalize_lut(const uint32_t* hist, uint32_t total, uint8_t* lut) {
    uint32_t cdf[256];
    cdf[0] = hist[0];
    for (int i = 1; i < 256; ++i) cdf[i] = cdf[i - 1] + hist[i];
    uint32_t cdf_min = 0;
    for (int i = 0; i < 256; ++i)
        if (cdf[i] > 0) { cdf_min = cdf[i]; break; }
    const uint32_t denominator = total - cdf_min;
    for (int i = 0; i < 256; ++i) {
        if (denominator == 0) lut[i] = (uint8_t)i;
        else if (cdf[i] >= cdf_min) lut[i] = (uint8_t)(((uint64_t)(cdf[i] - cdf_min) * 255u) / denominator);
        else lut[i] = 0;
    }
}

static bool hist_fmt(int pixfmt) { return pixfmt == ZO_PIX_U8 || pixfmt == ZO_PIX_RGB8 || pixfmt == ZO_PIX_RGBA8; }

// binary.zig:126-146 applyMorph, one pass
static void apply_morph(const std::vector<uint8_t>& src, std::vector<uint8_t>& dst, size_t rows, size_t cols, const uint8_t* kernel,
                        uint32_t kr_n, uint32_t kc_n, bool erode) {
    const int64_t anchor_r = kr_n / 2, anchor_c = kc_n / 2;
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) {
            uint8_t value = erode ? 255 : 0;
            bool done = false;
            for (uint32_t kr = 0; kr < kr_n && !done; ++kr) {
                const int64_t sr = (int64_t)r + kr - anchor_r;
                for (uint32_t kc = 0; kc < kc_n; ++kc) {
                    if (kernel[kr * kc_n + kc] == 0) continue;
                    const int64_t sc = (int64_t)c + kc - anchor_c;
                    const bool inside = sr >= 0 && sr < (int64_t)rows && sc >= 0 && sc < (int64_t)cols;   // atOrNull
                    const bool on = inside && src[(size_t)sr * cols + (size_t)sc] != 0;
                    if (!erode && on) { value = 255; done = true; break; }
                    if (erode && !on) { value = 0; done = true; break; }   // out of bounds is background
                }
            }
            dst[r * cols + c] = value;
        }
}

// binary.zig:183-224 morph: `iterations` passes (the temp / out ping-pong there only decides which buffer holds the result)
static void morph(std::vector<uint8_t>& img, size_t rows, size_t cols, const uint8_t* kernel, uint32_t kh, uint32_t kw, uint32_t iterations,
                  bool erode) {
    std::vector<uint8_t> tmp(img.size());
    for (uint32_t i = 0; i < iterations; ++i) {
        apply_morph(img, tmp, rows, cols, kernel, kh, kw, erode);
        img.swap(tmp);
    }
}

}  // namespace zo

using namespace zo;

extern "C" {

int zo_histogram(const zo_image* src, int pixfmt, uint32_t* counts) {
    if (!hist_fmt(pixfmt)) return ZO_ERR_UNSUPPORTED;
    histogram(src, channels_of(pixfmt), counts);
    return ZO_OK;
}

int zo_autocontrast(zo_image* img, int pixfmt, float cutoff) {
    if (!hist_fmt(pixfmt)) return ZO_ERR_UNSUPPORTED;
    if (!(cutoff >= 0.0f && cutoff < 0.5f)) return ZO_ERR_INVALID_CUTOFF;   // enhancement.zig:16-18 (NaN: no defined result there)
    const int ch = channels_of(pixfmt);
    const size_t total_pixels = (size_t)img->rows * img->cols;
    const uint32_t cutoff_pixels = (uint32_t)std::trunc((float)total_pixels * cutoff);   // :21
    uint32_t counts[4 * 256];
    histogram(img, ch, counts);
    uint8_t mins[4], maxs[4];
    for (int k = 0; k < ch; ++k) {
        mins[k] = find_cutoff_min(counts + 256 * k, cutoff_pixels);
        maxs[k] = find_cutoff_max(counts + 256 * k, cutoff_pixels);
    }
    uint8_t* base = (uint8_t*)img->data;
    const int remapped = ch == 4 ? 3 : ch;   // r, g, b only (:65-67): alpha untouched
    for (size_t r = 0; r < img->rows; ++r)
        for (size_t c = 0; c < img->cols; ++c)
            for (int k = 0; k < remapped; ++k) {
                uint8_t& v = base[(r * img->stride + c) * ch + k];
                v = remap(v, mins[k], maxs[k]);
            }
    return ZO_OK;
}

int zo_equalize(zo_image* img, int pixfmt) {
    if (!hist_fmt(pixfmt)) return ZO_ERR_UNSUPPORTED;
    const int ch = channels_of(pixfmt);
    const uint32_t total = (uint32_t)((size_t)img->rows * img->cols);   // enhancement.zig:85
    uint32_t counts[4 * 256];
    histogram(img, ch, counts);
    uint8_t lut[4 * 256];
    for (int k = 0; k < ch; ++k) equalize_lut(counts + 256 * k, total, lut + 256 * k);   // every channel, Rgba alpha too (:222-224)
    uint8_t* base = (uint8_t*)img->data;
    for (size_t r = 0; r < img->rows; ++r)
        for (size_t c = 0; c < img->cols; ++c)
            for (int k = 0; k < ch; ++k) {
                uint8_t& v = base[(r * img->stride + c) * ch + k];
                v = lut[256 * k + v];
            }
    return ZO_OK;
}

// binary.zig:38-84 (after image.zig:849 DimensionMismatch)
int zo_threshold_otsu(const zo_image* src, zo_image* dst, uint8_t* threshold_out) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;
    if (src->rows == 0 || src->cols == 0) { *threshold_out = 0; return ZO_OK; }
    uint32_t hist[256];
    histogram(src, 1, hist);
    const double total_pixels = (double)((size_t)src->rows * src->cols);
    double sum_total = 0;
    for (int i = 0; i < 256; ++i) sum_total += (double)hist[i] * (double)i;
    double sum_background = 0, weight_background = 0, max_variance = -1;
    uint8_t threshold = 0;
    for (int i = 0; i < 256; ++i) {
        const double count_f = (double)hist[i];
        weight_background += count_f;
        if (weight_background == 0) continue;
        const double weight_foreground = total_pixels - weight_background;
        if (weight_foreground == 0) break;
        sum_background += count_f * (double)i;
        const double mean_background = sum_background / weight_background;
        const double mean_foreground = (sum_total - sum_background) / weight_foreground;
        const double diff = mean_background - mean_foreground;
        const double variance = weight_background * weight_foreground * diff * diff;
        if (variance > max_variance) {
            max_variance = variance;
            threshold = (uint8_t)i;
        }
    }
    std::vector<uint8_t> in((size_t)src->rows * src->cols);   // src may alias dst
    for (size_t r = 0; r < src->rows; ++r)
        for (size_t c = 0; c < src->cols; ++c) in[r * src->cols + c] = ((const uint8_t*)src->data)[r * src->stride + c];
    for (size_t r = 0; r < src->rows; ++r)
        for (size_t c = 0; c < src->cols; ++c) ((uint8_t*)dst->data)[r * dst->stride + c] = in[r * src->cols + c] > threshold ? 255 : 0;
    *threshold_out = threshold;
    return ZO_OK;
}

// binary.zig:86-119 (after image.zig:862 DimensionMismatch): Integral.compute of the u8 plane, Integral.sum over the clipped window
int zo_threshold_adaptive_mean(const zo_image* src, zo_image* dst, uint32_t radius, float c) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;
    if (radius == 0) return ZO_ERR_INVALID_RADIUS;
    if (src->rows == 0 || src->cols == 0) return ZO_OK;
    const size_t rows = src->rows, cols = src->cols;
    std::vector<float> sat(rows * cols);
    integral_plane_u8(src, sat.data());
    std::vector<uint8_t> out(rows * cols);
    for (size_t row = 0; row < rows; ++row) {
        const size_t r1 = row > radius ? row - radius : 0, r2 = std::min(row + radius, rows - 1);
        for (size_t col = 0; col < cols; ++col) {
            const size_t c1 = col > radius ? col - radius : 0, c2 = std::min(col + radius, cols - 1);
            const float area = (float)((r2 - r1 + 1) * (c2 - c1 + 1));
            const float sum = sat[r2 * cols + c2] - (c1 > 0 ? sat[r2 * cols + (c1 - 1)] : 0.0f) - (r1 > 0 ? sat[(r1 - 1) * cols + c2] : 0.0f) +
                              ((r1 > 0 && c1 > 0) ? sat[(r1 - 1) * cols + (c1 - 1)] : 0.0f);   // integral.zig:86-89
            const float mean = sum / area;
            const float src_val = (float)((const uint8_t*)src->data)[row * src->stride + col];
            out[row * cols + col] = src_val > mean - c ? 255 : 0;
        }
    }
    for (size_t r = 0; r < rows; ++r)
        for (size_t col = 0; col < cols; ++col) ((uint8_t*)dst->data)[r * dst->stride + col] = out[r * cols + col];
    return ZO_OK;
}

// image.zig:870-914, binary.zig:9-33 (Kernel.init), :148-224.  op: ZO_MORPH_DILATE / ERODE / OPEN / CLOSE.
int zo_morph_binary(const zo_image* src, zo_image* dst, const uint8_t* kernel, uint32_t kernel_rows, uint32_t kernel_cols,
                    uint32_t iterations, int op) {
    if (kernel_rows == 0 || kernel_cols == 0 || kernel_rows % 2 == 0 || kernel_cols % 2 == 0) return ZO_ERR_INVALID_KERNEL_SIZE;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;
    const size_t rows = src->rows, cols = src->cols;
    const bool composite = op == ZO_MORPH_OPEN || op == ZO_MORPH_CLOSE;
    std::vector<uint8_t> img(rows * cols);
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) img[r * cols + c] = ((const uint8_t*)src->data)[r * src->stride + c];
    if (!(composite && iterations == 0)) {   // :170 copy
        if (rows == 0 || cols == 0) return ZO_OK;   // :190
        if (iterations > 0) {                       // :194 copy otherwise
            const bool first_erode = op == ZO_MORPH_ERODE || op == ZO_MORPH_OPEN;
            morph(img, rows, cols, kernel, kernel_rows, kernel_cols, iterations, first_erode);
            if (composite) morph(img, rows, cols, kernel, kernel_rows, kernel_cols, iterations, !first_erode);
        }
    }
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) ((uint8_t*)dst->data)[r * dst->stride + c] = img[r * cols + c];
    return ZO_OK;
}

}  // extern "C"
