// zo_visual.cpp -- CPU oracle of Image.diff (image/diff.zig:27-203 with stats.zig RunningStats), Image.applyColormap (image.zig:1190-1247,
// image/colormaps.zig:43-190), flipLeftRight / flipTopBottom (image/transforms.zig:28-45) and invert (image.zig:494-511, color.zig:328,441).
// TEST INFRASTRUCTURE ONLY (see zignal_oracle.h).  One thread, the reference's loops and operation order, -ffp-contract=off.
//
// Zig's @min / @max on floats return the non-NaN operand (zo_common.h zig_min / zig_max), so RunningStats' extrema skip a NaN sample
// while its sum and Welford moments take it, and std.math.clamp(NaN, lo, hi) = @max(lo, @min(NaN, hi)) = hi: meta.clamp(u8, NaN) is
// 255 and normalize's clamp of a NaN quotient is 1.
//
// The viridis and inferno tables are data in the reference; like the library, this oracle takes every table as an argument and only
// evaluates jet, heat and turbo itself.  Built on its own into oracle/libzo_visual.so (Makefile).
#include <cmath>
#include <cstring>

#include "zo_common.h"

extern "C" {
int zo_diff(const zo_image* a, const zo_image* b, zo_image* out, int pixfmt, float threshold, float scale, int binary, int force_opaque,
            double* stats7);
int zo_colormap_lut(int map, uint8_t* lut768);
int zo_apply_colormap(const zo_image* src, int pixfmt, const uint8_t* lut768, int has_min, double min, int has_max, double max,
                      zo_image* dst);
int zo_flip_left_right(zo_image* img, int pixfmt);
int zo_flip_top_bottom(zo_image* img, int pixfmt);
int zo_invert(zo_image* img, int pixfmt);
}

namespace zo {
namespace {

// RunningStats(f64, .summary): stats.zig:61-72 init, :80-105 add, :113-178 accessors.
struct RunningStats {
    uint64_t n = 0;
    double sum = 0, m1 = 0, m2 = 0;
    double min_val = INFINITY, max_val = -INFINITY;
    void add(double val) {
        const double n_ = (double)n;
        const double n1 = n_ + 1;
        const double delta = val - m1;
        const double delta_n = delta / n1;
        const double term1 = delta * delta_n * n_;
        m1 += delta_n;
        m2 += term1;
        sum += val;
        n += 1;
        min_val = zig_min(min_val, val);
        max_val = zig_max(max_val, val);
    }
    double mean() const { return n == 0 ? 0 : m1; }
    double variance() const { return n <= 1 ? 0 : m2 / (double)(n - 1); }
    double min() const { return n == 0 ? 0 : min_val; }
    double max() const { return n == 0 ? 0 : max_val; }
};

uint8_t* px_ptr(const zo_image* im, size_t r, size_t c, size_t pb) { return (uint8_t*)im->data + (r * im->stride + c) * pb; }

// diff.zig:41-143 for one pixel of N components of type CT.
template <typename CT, int N>
void diff_pixel(const CT* p1, const CT* p2, CT* dest, float threshold, float scale, bool binary, bool force_opaque, RunningStats& stats,
                uint64_t& diff_count) {
    constexpr bool flt = sizeof(CT) == 4;
    const CT max_v = flt ? (CT)1.0f : (CT)255;
    if (N == 1) {
        float d;
        if (flt) d = std::fabs((float)p1[0] - (float)p2[0]);                                        // :66
        else d = (float)(p1[0] > p2[0] ? p1[0] - p2[0] : p2[0] - p1[0]);                             // :49-50
        if (d > threshold) diff_count += 1;
        CT v = 0;
        if (binary) v = d > threshold ? max_v : (CT)0;
        else if (flt) v = (CT)(d * scale);
        else v = (CT)clamp_u8(d * scale);                                                           // meta.clamp(T, f32)
        dest[0] = v;
        stats.add((double)v);
        return;
    }
    bool is_pixel_diff = false;                                                                     // :81-99
    double pixel_max_val = 0;
    float diffs[N];
    for (int i = 0; i < N; ++i) {
        if (flt) diffs[i] = std::fabs((float)p1[i] - (float)p2[i]);
        else diffs[i] = (float)(p1[i] > p2[i] ? p1[i] - p2[i] : p2[i] - p1[i]);
        if (diffs[i] > threshold) is_pixel_diff = true;
    }
    if (is_pixel_diff) diff_count += 1;
    for (int i = 0; i < N; ++i) {                                                                   // :102-141
        const bool is_alpha = N == 4 && i == 3;
        if (force_opaque && is_alpha) {
            dest[i] = max_v;
        } else if (binary) {
            const CT val = is_pixel_diff ? max_v : (CT)0;
            dest[i] = val;
            if ((double)val > pixel_max_val) pixel_max_val = (double)val;
        } else {
            const float scaled = diffs[i] * scale;
            const CT val_out = flt ? (CT)scaled : (CT)clamp_u8(scaled);
            dest[i] = val_out;
            if ((double)val_out > pixel_max_val) pixel_max_val = (double)val_out;
        }
    }
    stats.add(pixel_max_val);
}

template <typename CT, int N>
void diff_image(const zo_image* a, const zo_image* b, zo_image* out, float threshold, float scale, bool binary, bool force_opaque,
                RunningStats& stats, uint64_t& diff_count) {
    const size_t pb = sizeof(CT) * N;
    for (size_t r = 0; r < a->rows; ++r)
        for (size_t c = 0; c < a->cols; ++c) {
            CT p1[N], p2[N];                                                                        // :43-44 copies: out may alias
            memcpy(p1, px_ptr(a, r, c, pb), pb);
            memcpy(p2, px_ptr(b, r, c, pb), pb);
            diff_pixel<CT, N>(p1, p2, (CT*)px_ptr(out, r, c, pb), threshold, scale, binary, force_opaque, stats, diff_count);
        }
}

// colormaps.zig:92-190, f64.
uint8_t round_u8(double v) { return (uint8_t)std::round(v); }

void jet_eval(double t, uint8_t* out) {
    const double gray = 8.0 * t;
    const double s = 1.0 / 2.0;
    uint8_t r = 0, g = 0, b = 0;
    if (gray <= 1) {
        r = 0; g = 0; b = round_u8((gray + 1) * s * 255.0);
    } else if (gray <= 3) {
        r = 0; g = round_u8((gray - 1) * s * 255.0); b = 255;
    } else if (gray <= 5) {
        r = round_u8((gray - 3) * s * 255.0); g = 255; b = round_u8((5 - gray) * s * 255.0);
    } else if (gray <= 7) {
        r = 255; g = round_u8((7 - gray) * s * 255.0); b = 0;
    } else {
        r = round_u8((9 - gray) * s * 255.0); g = 0; b = 0;
    }
    out[0] = r; out[1] = g; out[2] = b;
}

void heat_eval(double t, uint8_t* out) {
    const uint8_t r = round_u8(zig_min(t / 0.4, 1.0) * 255.0);
    uint8_t g = 0, b = 0;
    if (t > 0.4) g = round_u8(zig_min((t - 0.4) / 0.4, 1.0) * 255.0);
    if (t > 0.8) b = round_u8(zig_min((t - 0.8) / 0.2, 1.0) * 255.0);
    out[0] = r; out[1] = g; out[2] = b;
}

void turbo_eval(double t, uint8_t* out) {
    const double r_coeffs[6] = {0.13572138, 4.61539260, -42.66032258, 132.13108234, -152.94239396, 59.28637943};
    const double g_coeffs[6] = {0.09140261, 2.19418839, 4.84296658, -14.18503333, 4.27729857, 2.82956604};
    const double b_coeffs[6] = {0.10667330, 12.64194608, -60.58204836, 110.36276771, -89.90310912, 27.34824973};
    const double t2 = t * t;
    const double t3 = t2 * t;
    const double t4 = t3 * t;
    const double t5 = t4 * t;
    const double v[6] = {1.0, t, t2, t3, t4, t5};
    const double* coeffs[3] = {r_coeffs, g_coeffs, b_coeffs};
    for (int ch = 0; ch < 3; ++ch) {
        double prod[6];
        for (int k = 0; k < 6; ++k) prod[k] = v[k] * coeffs[ch][k];                                 // v * coeffs
        double acc = prod[0];                                                                       // @reduce(.Add), left to right
        for (int k = 1; k < 6; ++k) acc = acc + prod[k];
        out[ch] = round_u8(zig_max(0.0, zig_min(acc, 1.0)) * 255.0);                               // math.clamp(v, 0, 1)
    }
}

// meta.zig:255-260
double normalize(double value, double min, double max) {
    if (std::isnan(value) || std::isnan(min) || std::isnan(max)) return 0;
    if (max <= min) return 0;
    return zig_max(0.0, zig_min((value - min) / (max - min), 1.0));
}

inline uint8_t luma_u8(uint8_t r, uint8_t g, uint8_t b) {                                           // rgbToGray(u8), color.zig:1031-1041
    const int y = (13933 * (int)r + 46871 * (int)g + 4732 * (int)b + 32768) >> 16;
    return (uint8_t)(y < 0 ? 0 : (y > 255 ? 255 : y));
}

// image.zig:1217 / :1239: meta.as(f64, px) for scalars, convertColor(f64, px) = px.to(.gray).as(f64).y for colours.
double pixel_value(const uint8_t* p, int pixfmt) {
    switch (pixfmt) {
        case ZO_PIX_U8: return (double)p[0];
        case ZO_PIX_F32: { float f; memcpy(&f, p, 4); return (double)f; }
        case ZO_PIX_RGB8: case ZO_PIX_RGBA8: return (double)luma_u8(p[0], p[1], p[2]) / 255.0;     // Gray(u8).as(f64): y / 255
        default: {
            float f[4];
            memcpy(f, p, 16);
            const float l = 0.2126f * f[0] + 0.7152f * f[1] + 0.0722f * f[2];                        // rgbToGray(f32), color.zig:1043-1045
            const float c = zig_max(0.0f, zig_min(l, 1.0f));
            return (double)c;                                                                       // Gray(f32).as(f64): @floatCast
        }
    }
}

}  // namespace
}  // namespace zo

using namespace zo;

extern "C" int zo_diff(const zo_image* a, const zo_image* b, zo_image* out, int pixfmt, float threshold, float scale, int binary,
                       int force_opaque, double* stats7) {
    if (a->rows != b->rows || a->cols != b->cols || a->rows != out->rows || a->cols != out->cols) return 1;
    RunningStats stats;
    uint64_t diff_count = 0;
    switch (pixfmt) {
        case ZO_PIX_U8: diff_image<uint8_t, 1>(a, b, out, threshold, scale, binary, force_opaque, stats, diff_count); break;
        case ZO_PIX_F32: diff_image<float, 1>(a, b, out, threshold, scale, binary, force_opaque, stats, diff_count); break;
        case ZO_PIX_RGB8: diff_image<uint8_t, 3>(a, b, out, threshold, scale, binary, force_opaque, stats, diff_count); break;
        case ZO_PIX_RGBA8: diff_image<uint8_t, 4>(a, b, out, threshold, scale, binary, force_opaque, stats, diff_count); break;
        case ZO_PIX_RGBAF32: diff_image<float, 4>(a, b, out, threshold, scale, binary, force_opaque, stats, diff_count); break;
        default: return 3;
    }
    stats7[0] = (double)stats.n;
    stats7[1] = (double)diff_count;
    stats7[2] = stats.sum;
    stats7[3] = stats.mean();
    stats7[4] = stats.variance();
    stats7[5] = stats.min();
    stats7[6] = stats.max();
    return 0;
}

extern "C" int zo_colormap_lut(int map, uint8_t* lut768) {
    for (int i = 0; i < 256; ++i) {                                                                 // colormaps.zig:124-131 and the like
        const double t = (double)i / 255.0;
        if (map == 0) jet_eval(t, lut768 + 3 * i);
        else if (map == 1) heat_eval(t, lut768 + 3 * i);
        else if (map == 2) turbo_eval(t, lut768 + 3 * i);
        else return 3;
    }
    return 0;
}

extern "C" int zo_apply_colormap(const zo_image* src, int pixfmt, const uint8_t* lut768, int has_min, double min, int has_max, double max,
                                 zo_image* dst) {
    const size_t pb = pixel_bytes(pixfmt);
    double min_val = 0, max_val = 0;                                                                // image.zig:1198-1233
    if (!has_min || !has_max) {
        double min_v = std::numeric_limits<double>::max();
        double max_v = -std::numeric_limits<double>::max();
        if ((size_t)src->rows * src->cols == 0) {
            min_v = 0;
            max_v = 1;
        } else {
            for (size_t r = 0; r < src->rows; ++r)
                for (size_t c = 0; c < src->cols; ++c) {
                    const double val = pixel_value(px_ptr(src, r, c, pb), pixfmt);
                    min_v = zig_min(min_v, val);
                    max_v = zig_max(max_v, val);
                }
        }
        min_val = has_min ? min : min_v;
        max_val = has_max ? max : max_v;
    } else {
        min_val = min;
        max_val = max;
    }
    if (max_val <= min_val) max_val = min_val + 1.0;
    for (size_t r = 0; r < src->rows; ++r)                                                          // :1237-1245, colormaps.zig:45-49
        for (size_t c = 0; c < src->cols; ++c) {
            const double val = pixel_value(px_ptr(src, r, c, pb), pixfmt);
            const double t = normalize(val, min_val, max_val);
            const size_t index = (size_t)std::round(t * 255.0);
            memcpy(px_ptr(dst, r, c, 3), lut768 + 3 * index, 3);
        }
    return 0;
}

extern "C" int zo_flip_left_right(zo_image* img, int pixfmt) {                                      // transforms.zig:28-33 (std.mem.reverse)
    const size_t pb = pixel_bytes(pixfmt);
    uint8_t tmp[16];
    for (size_t r = 0; r < img->rows; ++r)
        for (size_t i = 0, j = img->cols; i + 1 < j; ++i, --j) {
            uint8_t *x = px_ptr(img, r, i, pb), *y = px_ptr(img, r, j - 1, pb);
            memcpy(tmp, x, pb); memcpy(x, y, pb); memcpy(y, tmp, pb);
        }
    return 0;
}

extern "C" int zo_flip_top_bottom(zo_image* img, int pixfmt) {                                      // transforms.zig:36-44
    const size_t pb = pixel_bytes(pixfmt);
    uint8_t tmp[16];
    for (size_t r = 0; r < img->rows / 2; ++r)
        for (size_t c = 0; c < img->cols; ++c) {
            uint8_t *t = px_ptr(img, r, c, pb), *b = px_ptr(img, img->rows - r - 1, c, pb);
            memcpy(tmp, t, pb); memcpy(t, b, pb); memcpy(b, tmp, pb);
        }
    return 0;
}

extern "C" int zo_invert(zo_image* img, int pixfmt) {                                               // image.zig:494-511
    if (pixfmt == ZO_PIX_F32) return 3;                                                             // no invert() on f32: compile error
    const size_t pb = pixel_bytes(pixfmt);
    for (size_t r = 0; r < img->rows; ++r)
        for (size_t c = 0; c < img->cols; ++c) {
            uint8_t* p = px_ptr(img, r, c, pb);
            if (pixfmt == ZO_PIX_RGBAF32) {                                                         // Rgba(f32).invert: 1.0 - c, alpha kept
                float f[4];
                memcpy(f, p, 16);
                for (int k = 0; k < 3; ++k) f[k] = 1.0f - f[k];
                memcpy(p, f, 16);
            } else {
                const int n = pixfmt == ZO_PIX_U8 ? 1 : 3;                                          // 255 - v; Rgba(u8) alpha kept
                for (int k = 0; k < n; ++k) p[k] = (uint8_t)(255 - p[k]);
            }
        }
    return 0;
}
