// zo_conv.cpp -- CPU oracle for Image.convolve / convolveSeparable / gaussianBlur.
// TEST INFRASTRUCTURE ONLY (see zignal_oracle.h).  Restates, line by line:
//   image/convolution.zig:18-22 (divClampU8), :76-195 (ConvolutionKernel), :198-301 (convolve),
//   :303-309 (scaleKernelToInt), :313-438 (convolveSeparable), :441-647 (convolveSeparablePlane),
//   :650-655 (getPixel), image.zig:954-994 (gaussianBlur), border.zig:32-63.
// Build with -ffp-contract=off: the reference never fuses mul+add (no @mulAdd on this path).
#include <omp.h>

#include "zo_common.h"

namespace zo {

int g_threads = 1;

// convolution.zig:650-655 getPixel: border-resolved read, 0 when resolveIndex says null.
template <typename T, typename R>
static inline R get_pixel(const Img<T>& img, int64_t row, int64_t col, int border) {
    const int64_t r = resolve_index(row, (int64_t)img.rows, border);
    if (r < 0) return (R)0;
    const int64_t c = resolve_index(col, (int64_t)img.cols, border);
    if (c < 0) return (R)0;
    return (R)img.at((size_t)r, (size_t)c);
}

static constexpr int kVecLenF32 = 8;   // std.simd.suggestVectorLength(f32) on AVX2; only shapes loops
static constexpr int kVecLenI32 = 8;

// ---------------------------------------------------------------------------------------------
// convolveSeparablePlane, f32 instance (PixelT = TempT = AccumT = f32): convolution.zig:441-647
// ---------------------------------------------------------------------------------------------
static void conv_sep_plane_f32(const Img<float>& src, const Img<float>& dst, const Img<float>& tmp,
                               const float* kx, size_t nx, const float* ky, size_t ny, int border) {
    const size_t half_x = nx / 2, half_y = ny / 2;
    const size_t rows = src.rows, cols = src.cols;
    auto negligible = [](float k) { return std::fabs(k) < 1e-10f; };  // :459-467
    constexpr size_t VL = kVecLenF32;

    // Horizontal pass (src -> temp), :516-576
#pragma omp parallel for schedule(static) num_threads(g_threads) if (g_threads > 1)
    for (size_t r = 0; r < rows; ++r) {
        const float* srow = src.data + r * src.stride;
        float* trow = tmp.data + r * tmp.stride;
        size_t c = 0;
        const size_t left_border_end = std::min(half_x, cols);
        for (; c < left_border_end; ++c) {  // :523-532 (no negligible skip here)
            float result = 0;
            for (size_t i = 0; i < nx; ++i) {
                const int64_t icx = (int64_t)c + (int64_t)i - (int64_t)half_x;
                const float pv = get_pixel<float, float>(src, (int64_t)r, icx, border);
                result += pv * kx[i];
            }
            trow[c] = result;
        }
        if (cols > 2 * half_x) {
            const size_t interior_end = cols - half_x;
            for (; c + VL <= interior_end; c += VL) {  // :537-551
                float acc[VL];
                for (size_t l = 0; l < VL; ++l) acc[l] = 0;
                for (size_t ki = 0; ki < nx; ++ki) {
                    const float k = kx[ki];
                    if (!negligible(k)) {
                        const float* s = srow + c + ki - half_x;
                        for (size_t l = 0; l < VL; ++l) acc[l] += s[l] * k;
                    }
                }
                for (size_t l = 0; l < VL; ++l) trow[c + l] = acc[l];
            }
            for (; c < interior_end; ++c) {  // :553-563
                float result = 0;
                const size_t c0 = c - half_x;
                for (size_t i = 0; i < nx; ++i) {
                    const float k = kx[i];
                    if (!negligible(k)) result += srow[c0 + i] * k;
                }
                trow[c] = result;
            }
        }
        for (; c < cols; ++c) {  // :566-575
            float result = 0;
            for (size_t i = 0; i < nx; ++i) {
                const int64_t icx = (int64_t)c + (int64_t)i - (int64_t)half_x;
                const float pv = get_pixel<float, float>(src, (int64_t)r, icx, border);
                result += pv * kx[i];
            }
            trow[c] = result;
        }
    }

    // Vertical pass (temp -> dst), 16-column tiles, :578-623
    const size_t tile_width = std::max<size_t>(VL, 16);
    if (rows > 2 * half_y) {
        const size_t safe_end_r = rows - half_y;
        const size_t ntiles = (cols + tile_width - 1) / tile_width;
#pragma omp parallel for schedule(static) num_threads(g_threads) if (g_threads > 1)
        for (size_t t = 0; t < ntiles; ++t) {
            const size_t tile_c = t * tile_width;
            const size_t tile_end = std::min(tile_c + tile_width, cols);
            size_t c = tile_c;
            for (; c + VL <= tile_end; c += VL) {
                for (size_t r = half_y; r < safe_end_r; ++r) {
                    float acc[VL];
                    for (size_t l = 0; l < VL; ++l) acc[l] = 0;
                    for (size_t ki = 0; ki < ny; ++ki) {
                        const float k = ky[ki];
                        if (!negligible(k)) {
                            const float* s = tmp.data + (r + ki - half_y) * tmp.stride + c;
                            for (size_t l = 0; l < VL; ++l) acc[l] += s[l] * k;
                        }
                    }
                    float* d = dst.data + r * dst.stride + c;
                    for (size_t l = 0; l < VL; ++l) d[l] = acc[l];
                }
            }
            for (; c < tile_end; ++c) {  // :609-621
                for (size_t r = half_y; r < safe_end_r; ++r) {
                    float result = 0;
                    const size_t r0 = r - half_y;
                    for (size_t i = 0; i < ny; ++i) {
                        const float k = ky[i];
                        if (negligible(k)) continue;
                        result += tmp.data[(r0 + i) * tmp.stride + c] * k;
                    }
                    dst.data[r * dst.stride + c] = result;
                }
            }
        }
    }

    // Top and bottom border rows, :625-646 (getPixel on temp; no negligible skip)
    const size_t top_end = std::min(half_y, rows);
    const size_t bottom_start = (rows > half_y) ? std::max(top_end, rows - half_y) : rows;
    const size_t ranges[2][2] = {{0, top_end}, {bottom_start, rows}};
    for (auto& range : ranges) {
        for (size_t r = range[0]; r < range[1]; ++r) {
            for (size_t c = 0; c < cols; ++c) {
                float result = 0;
                for (size_t i = 0; i < ny; ++i) {
                    const int64_t iry = (int64_t)r + (int64_t)i - (int64_t)half_y;
                    const float pv = get_pixel<float, float>(tmp, iry, (int64_t)c, border);
                    result += pv * ky[i];
                }
                dst.data[r * dst.stride + c] = result;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// convolveSeparablePlane, u8 instance (PixelT = u8, TempT = i32, AccumT = i64): :441-647
// ---------------------------------------------------------------------------------------------
static void conv_sep_plane_u8(const Img<uint8_t>& src, const Img<uint8_t>& dst, const Img<int32_t>& tmp,
                              const int32_t* kx, size_t nx, const int32_t* ky, size_t ny, int border) {
    const size_t half_x = nx / 2, half_y = ny / 2;
    const size_t rows = src.rows, cols = src.cols;
    constexpr size_t VL = kVecLenI32;
    constexpr int64_t SCALE_SQ = 65536;  // fixed_point_scale_sq, :15
    auto store_temp = [](int64_t v) { return clamp_from_int<int32_t>(v); };  // :507-513

#pragma omp parallel for schedule(static) num_threads(g_threads) if (g_threads > 1)
    for (size_t r = 0; r < rows; ++r) {
        const uint8_t* srow = src.data + r * src.stride;
        int32_t* trow = tmp.data + r * tmp.stride;
        size_t c = 0;
        const size_t left_border_end = std::min(half_x, cols);
        for (; c < left_border_end; ++c) {
            int64_t result = 0;
            for (size_t i = 0; i < nx; ++i) {
                const int64_t icx = (int64_t)c + (int64_t)i - (int64_t)half_x;
                const int32_t pv = get_pixel<uint8_t, int32_t>(src, (int64_t)r, icx, border);
                result += (int64_t)pv * (int64_t)kx[i];
            }
            trow[c] = store_temp(result);
        }
        if (cols > 2 * half_x) {
            const size_t interior_end = cols - half_x;
            for (; c + VL <= interior_end; c += VL) {
                int64_t acc[VL];
                for (size_t l = 0; l < VL; ++l) acc[l] = 0;
                for (size_t ki = 0; ki < nx; ++ki) {
                    const int64_t k = kx[ki];
                    if (k != 0) {
                        const uint8_t* s = srow + c + ki - half_x;
                        for (size_t l = 0; l < VL; ++l) acc[l] += (int64_t)s[l] * k;
                    }
                }
                for (size_t l = 0; l < VL; ++l) trow[c + l] = store_temp(acc[l]);
            }
            for (; c < interior_end; ++c) {
                int64_t result = 0;
                const size_t c0 = c - half_x;
                for (size_t i = 0; i < nx; ++i)
                    if (kx[i] != 0) result += (int64_t)srow[c0 + i] * (int64_t)kx[i];
                trow[c] = store_temp(result);
            }
        }
        for (; c < cols; ++c) {
            int64_t result = 0;
            for (size_t i = 0; i < nx; ++i) {
                const int64_t icx = (int64_t)c + (int64_t)i - (int64_t)half_x;
                const int32_t pv = get_pixel<uint8_t, int32_t>(src, (int64_t)r, icx, border);
                result += (int64_t)pv * (int64_t)kx[i];
            }
            trow[c] = store_temp(result);
        }
    }

    const size_t tile_width = std::max<size_t>(VL, 16);
    if (rows > 2 * half_y) {
        const size_t safe_end_r = rows - half_y;
        const size_t ntiles = (cols + tile_width - 1) / tile_width;
#pragma omp parallel for schedule(static) num_threads(g_threads) if (g_threads > 1)
        for (size_t t = 0; t < ntiles; ++t) {
            const size_t tile_c = t * tile_width;
            const size_t tile_end = std::min(tile_c + tile_width, cols);
            size_t c = tile_c;
            for (; c + VL <= tile_end; c += VL) {
                for (size_t r = half_y; r < safe_end_r; ++r) {
                    int64_t acc[VL];
                    for (size_t l = 0; l < VL; ++l) acc[l] = 0;
                    for (size_t ki = 0; ki < ny; ++ki) {
                        const int64_t k = ky[ki];
                        if (k != 0) {
                            const int32_t* s = tmp.data + (r + ki - half_y) * tmp.stride + c;
                            for (size_t l = 0; l < VL; ++l) acc[l] += (int64_t)s[l] * k;
                        }
                    }
                    uint8_t* d = dst.data + r * dst.stride + c;
                    for (size_t l = 0; l < VL; ++l) d[l] = div_clamp_u8(acc[l], SCALE_SQ);
                }
            }
            for (; c < tile_end; ++c) {
                for (size_t r = half_y; r < safe_end_r; ++r) {
                    int64_t result = 0;
                    const size_t r0 = r - half_y;
                    for (size_t i = 0; i < ny; ++i) {
                        if (ky[i] == 0) continue;
                        result += (int64_t)tmp.data[(r0 + i) * tmp.stride + c] * (int64_t)ky[i];
                    }
                    dst.data[r * dst.stride + c] = div_clamp_u8(result, SCALE_SQ);
                }
            }
        }
    }

    const size_t top_end = std::min(half_y, rows);
    const size_t bottom_start = (rows > half_y) ? std::max(top_end, rows - half_y) : rows;
    const size_t ranges[2][2] = {{0, top_end}, {bottom_start, rows}};
    for (auto& range : ranges) {
        for (size_t r = range[0]; r < range[1]; ++r) {
            for (size_t c = 0; c < cols; ++c) {
                int64_t result = 0;
                for (size_t i = 0; i < ny; ++i) {
                    const int64_t iry = (int64_t)r + (int64_t)i - (int64_t)half_y;
                    const int32_t pv = get_pixel<int32_t, int32_t>(tmp, iry, (int64_t)c, border);
                    result += (int64_t)pv * (int64_t)ky[i];
                }
                dst.data[r * dst.stride + c] = div_clamp_u8(result, SCALE_SQ);
            }
        }
    }
}

// convolution.zig:303-309 scaleKernelToInt
static std::vector<int32_t> scale_kernel_to_int(const float* k, size_t n, int scale) {
    std::vector<int32_t> out(n);
    for (size_t i = 0; i < n; ++i) out[i] = as_i32(k[i] * (float)scale);
    return out;
}

static inline bool preserves_uniform(int border) { return border != ZO_BORDER_ZERO; }  // border.zig:22-27

// convolution.zig:313-438 convolveSeparable
static int conv_separable(const zo_image* src, zo_image* dst, int pixfmt, const float* kx, int nx,
                          const float* ky, int ny, int border) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;  // image.zig:947
    if (nx <= 0 || ny <= 0) return ZO_ERR_INVALID_ARGUMENT;
    const uint32_t rows = src->rows, cols = src->cols;
    switch (pixfmt) {
        case ZO_PIX_U8: {  // :323-333
            Plane<int32_t> temp(rows, cols);
            auto kxi = scale_kernel_to_int(kx, nx, 256), kyi = scale_kernel_to_int(ky, ny, 256);
            conv_sep_plane_u8(Img<uint8_t>(src), Img<uint8_t>(dst), temp.img(), kxi.data(), nx, kyi.data(), ny, border);
            return ZO_OK;
        }
        case ZO_PIX_F32: {  // :334-339
            Plane<float> temp(rows, cols);
            conv_sep_plane_f32(Img<float>(src), Img<float>(dst), temp.img(), kx, nx, ky, ny, border);
            return ZO_OK;
        }
        case ZO_PIX_RGB8:
        case ZO_PIX_RGBA8: {  // :340-431
            const int ch = channels_of(pixfmt);
            const size_t plane_size = (size_t)rows * cols;
            auto kxi = scale_kernel_to_int(kx, nx, 256), kyi = scale_kernel_to_int(ky, ny, 256);
            int64_t kx_sum = 0, ky_sum = 0;
            for (auto w : kxi) kx_sum += w;
            for (auto w : kyi) ky_sum += w;
            const int64_t kernel_sum = kx_sum * ky_sum;
            const int64_t scale_sq = 65536;
            std::vector<std::vector<uint8_t>> channels;
            bool uniform[4];
            uint8_t uval[4];
            split_channels_u8(ch, (const uint8_t*)src->data, rows, cols, (size_t)src->stride, channels, uniform, uval);
            enum { NORMALIZED, SCALED, NON_UNIFORM } strategy[4];
            const bool safe = preserves_uniform(border);
            for (int i = 0; i < ch; ++i) {
                if (uniform[i] && safe) strategy[i] = (kernel_sum == scale_sq) ? NORMALIZED : SCALED;
                else strategy[i] = NON_UNIFORM;
            }
            std::vector<std::vector<uint8_t>> out_channels(ch);
            Plane<int32_t> temp(rows, cols);
            for (int i = 0; i < ch; ++i) {
                if (strategy[i] == NORMALIZED) continue;
                out_channels[i].resize(plane_size);
                if (strategy[i] == SCALED) {
                    const int64_t accum = (int64_t)uval[i] * kernel_sum;
                    std::fill(out_channels[i].begin(), out_channels[i].end(), div_clamp_u8(accum, scale_sq));
                }
            }
            for (int i = 0; i < ch; ++i) {
                if (strategy[i] != NON_UNIFORM) continue;
                Img<uint8_t> sp(channels[i].data(), rows, cols, cols), dp(out_channels[i].data(), rows, cols, cols);
                conv_sep_plane_u8(sp, dp, temp.img(), kxi.data(), nx, kyi.data(), ny, border);
            }
            const uint8_t* finals[4];
            for (int i = 0; i < ch; ++i)
                finals[i] = (strategy[i] == NORMALIZED) ? channels[i].data() : out_channels[i].data();
            merge_channels_u8(finals, ch, (uint8_t*)dst->data, rows, cols, (size_t)dst->stride);
            return ZO_OK;
        }
        case ZO_PIX_RGBAF32: {  // extension: per-channel Image(f32) planes (SURVEY.md 0.1 / 8a-5)
            Plane<float> sp(rows, cols), dp(rows, cols), temp(rows, cols);
            const float* s = (const float*)src->data;
            float* d = (float*)dst->data;
            for (int chn = 0; chn < 4; ++chn) {
                for (uint32_t r = 0; r < rows; ++r)
                    for (uint32_t c = 0; c < cols; ++c) sp.buf[(size_t)r * cols + c] = s[(r * src->stride + c) * 4 + chn];
                conv_sep_plane_f32(sp.img(), dp.img(), temp.img(), kx, nx, ky, ny, border);
                for (uint32_t r = 0; r < rows; ++r)
                    for (uint32_t c = 0; c < cols; ++c) d[(r * dst->stride + c) * 4 + chn] = dp.buf[(size_t)r * cols + c];
            }
            return ZO_OK;
        }
    }
    return ZO_ERR_UNSUPPORTED;
}

// ---------------------------------------------------------------------------------------------
// ConvolutionKernel(T, rows, cols).convolve: convolution.zig:113-193 (runtime kh, kw here).
// Every branch of the reference (border pixel, SIMD interior, scalar interior) accumulates
// `result += pixel * k` over taps in row-major order starting from 0, so they are one formula.
// ---------------------------------------------------------------------------------------------
template <typename T, typename KS, typename AS>
static void convolve_plane(const Img<T>& src, const Img<T>& dst, const KS* kernel, size_t kh, size_t kw, int border,
                           T (*store)(AS)) {
    const size_t half_h = kh / 2, half_w = kw / 2;
    const size_t rows = src.rows, cols = src.cols;
#pragma omp parallel for schedule(static) num_threads(g_threads) if (g_threads > 1)
    for (size_t r = 0; r < rows; ++r) {
        const bool row_in_band = r >= half_h && r + half_h < rows;  // :137
        for (size_t c = 0; c < cols; ++c) {
            AS result = 0;
            if (row_in_band && c >= half_w && c + half_w < cols) {  // :176-187 / :155-172
                for (size_t ky = 0; ky < kh; ++ky) {
                    const T* s = src.data + (r + ky - half_h) * src.stride + (c - half_w);
                    for (size_t kx = 0; kx < kw; ++kx) result += (AS)s[kx] * (AS)kernel[ky * kw + kx];
                }
            } else {  // :113-127 convolvePixelWithBorder
                for (size_t ky = 0; ky < kh; ++ky)
                    for (size_t kx = 0; kx < kw; ++kx) {
                        const int64_t iry = (int64_t)r + (int64_t)ky - (int64_t)half_h;
                        const int64_t icx = (int64_t)c + (int64_t)kx - (int64_t)half_w;
                        const AS pv = (AS)get_pixel<T, AS>(src, iry, icx, border);
                        result += pv * (AS)kernel[ky * kw + kx];
                    }
            }
            dst.data[r * dst.stride + c] = store(result);
        }
    }
}
static uint8_t store_u8_256(int64_t a) { return div_clamp_u8(a, 256); }  // PixelIO(u8).store, :62-64
static float store_f32(float a) { return a; }

// convolution.zig:198-301 convolve
static int convolve(const zo_image* src, zo_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;  // image.zig:927
    if (kh <= 0 || kw <= 0) return ZO_ERR_INVALID_ARGUMENT;
    const uint32_t rows = src->rows, cols = src->cols;
    const size_t size = (size_t)kh * kw;
    switch (pixfmt) {
        case ZO_PIX_F32:
            convolve_plane<float, float, float>(Img<float>(src), Img<float>(dst), kernel, kh, kw, border, store_f32);
            return ZO_OK;
        case ZO_PIX_U8: {
            std::vector<int32_t> ki(size);
            for (size_t i = 0; i < size; ++i) ki[i] = as_i32(kernel[i] * 256.0f);  // flatten, :94-111
            convolve_plane<uint8_t, int32_t, int64_t>(Img<uint8_t>(src), Img<uint8_t>(dst), ki.data(), kh, kw, border, store_u8_256);
            return ZO_OK;
        }
        case ZO_PIX_RGB8:
        case ZO_PIX_RGBA8: {  // :213-294
            const int ch = channels_of(pixfmt);
            std::vector<int32_t> ki(size);
            int32_t kernel_sum = 0;
            for (size_t i = 0; i < size; ++i) { ki[i] = as_i32(kernel[i] * 256.0f); kernel_sum += ki[i]; }
            const size_t plane_size = (size_t)rows * cols;
            std::vector<std::vector<uint8_t>> channels;
            bool uniform[4];
            uint8_t uval[4];
            split_channels_u8(ch, (const uint8_t*)src->data, rows, cols, (size_t)src->stride, channels, uniform, uval);
            enum { NORMALIZED, SCALED, NON_UNIFORM } strategy[4];
            const bool safe = preserves_uniform(border);
            for (int i = 0; i < ch; ++i) {
                if (uniform[i] && safe) strategy[i] = (kernel_sum == 256) ? NORMALIZED : SCALED;
                else strategy[i] = NON_UNIFORM;
            }
            std::vector<std::vector<uint8_t>> out_channels(ch);
            for (int i = 0; i < ch; ++i) {
                if (strategy[i] == NORMALIZED) continue;
                out_channels[i].resize(plane_size);
                if (strategy[i] == SCALED) {
                    const int64_t accum = (int64_t)uval[i] * (int64_t)kernel_sum;
                    std::fill(out_channels[i].begin(), out_channels[i].end(), store_u8_256(accum));
                }
            }
            for (int i = 0; i < ch; ++i) {
                if (strategy[i] != NON_UNIFORM) continue;
                Img<uint8_t> sp(channels[i].data(), rows, cols, cols), dp(out_channels[i].data(), rows, cols, cols);
                convolve_plane<uint8_t, int32_t, int64_t>(sp, dp, ki.data(), kh, kw, border, store_u8_256);
            }
            const uint8_t* finals[4];
            for (int i = 0; i < ch; ++i)
                finals[i] = (strategy[i] == NORMALIZED) ? channels[i].data() : out_channels[i].data();
            merge_channels_u8(finals, ch, (uint8_t*)dst->data, rows, cols, (size_t)dst->stride);
            return ZO_OK;
        }
    }
    return ZO_ERR_UNSUPPORTED;
}

// image.zig:375-392 copy (view-aware)
static void copy_image(const zo_image* src, zo_image* dst, int pixfmt) {
    if (src->data == dst->data) return;
    const size_t pb = pixel_bytes(pixfmt);
    for (uint32_t r = 0; r < src->rows; ++r)
        std::memcpy((uint8_t*)dst->data + r * dst->stride * pb, (const uint8_t*)src->data + r * src->stride * pb,
                    (size_t)src->cols * pb);
}

// image.zig:972-990
static int gaussian_taps(float sigma, float* taps, int cap) {
    if (sigma == 0) return 0;
    if (sigma < 0) return -1;
    const size_t radius = (size_t)std::ceil(3.0f * sigma);
    const size_t kernel_size = 2 * radius + 1;
    if ((size_t)cap < kernel_size) return -2;
    float sum = 0;
    for (size_t i = 0; i < kernel_size; ++i) {
        const float x = (float)i - (float)radius;
        taps[i] = std::exp(-(x * x) / (2.0f * sigma * sigma));  // @exp in f32
        sum += taps[i];
    }
    for (size_t i = 0; i < kernel_size; ++i) taps[i] /= sum;
    return (int)kernel_size;
}

}  // namespace zo

extern "C" {

void zo_set_threads(int n) { zo::g_threads = n < 1 ? 1 : n; }
int zo_get_threads(void) { return zo::g_threads; }
int zo_hw_threads(void) { return omp_get_num_procs(); }

// Benchmark helper (not a reference function): fill a rows x cols f32 plane with uniform [0, 1) values, rows split across the
// threads exactly like the row-parallel convolution loops (static schedule), so every page is first touched -- and therefore
// placed on the NUMA node of -- the thread that will later read and write it.
void zo_parallel_fill_f32(float* p, uint64_t rows, uint64_t cols, uint64_t seed) {
    const int g_threads = zo::g_threads;
#pragma omp parallel for schedule(static) num_threads(g_threads) if (g_threads > 1)
    for (int64_t r = 0; r < (int64_t)rows; ++r) {
        uint64_t x = seed * 0x9E3779B97F4A7C15ull + (uint64_t)r * 0xD1B54A32D192ED03ull + 1;
        float* row = p + (size_t)r * cols;
        for (uint64_t c = 0; c < cols; ++c) {
            x ^= x >> 12; x ^= x << 25; x ^= x >> 27;                       // xorshift64*
            row[c] = (float)((x * 0x2545F4914F6CDD1Dull) >> 40) * (1.0f / 16777216.0f);
        }
    }
}

int64_t zo_resolve_index(int64_t idx, int64_t length, int border) { return zo::resolve_index(idx, length, border); }
uint8_t zo_clamp_u8_f32(float v) { return zo::clamp_u8(v); }
uint8_t zo_div_clamp_u8(int64_t accum, int64_t scale) { return zo::div_clamp_u8(accum, scale); }

int zo_gaussian_taps(float sigma, float* taps, int cap) { return zo::gaussian_taps(sigma, taps, cap); }

int zo_conv_separable(const zo_image* src, zo_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny,
                      int border) {
    return zo::conv_separable(src, dst, pixfmt, kx, nx, ky, ny, border);
}

int zo_convolve(const zo_image* src, zo_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border) {
    return zo::convolve(src, dst, pixfmt, kernel, kh, kw, border);
}

// edges.zig:33-73 Edges(T).sobel: gray f32 (as(f32, convertColor(u8, px)); float scalars pass through), two 3x3 convolutions with
// .replicate, magnitude sqrt(gx^2 + gy^2) / 4, trunc(clamp(0, 255)) into a u8 image.  color.zig:1031-1041 for the luma.
int zo_sobel(const zo_image* src, zo_image* dst, int pixfmt) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;   // image.zig:1005
    const uint32_t rows = src->rows, cols = src->cols;
    std::vector<float> gray((size_t)rows * cols), gx((size_t)rows * cols), gy((size_t)rows * cols);
    for (uint32_t r = 0; r < rows; ++r)
        for (uint32_t c = 0; c < cols; ++c) {
            float v;
            if (pixfmt == ZO_PIX_F32) {
                v = ((const float*)src->data)[(size_t)r * src->stride + c];
            } else if (pixfmt == ZO_PIX_U8) {
                v = (float)((const uint8_t*)src->data)[(size_t)r * src->stride + c];
            } else if (pixfmt == ZO_PIX_RGB8 || pixfmt == ZO_PIX_RGBA8) {
                const int ch = pixfmt == ZO_PIX_RGB8 ? 3 : 4;
                const uint8_t* px = (const uint8_t*)src->data + ((size_t)r * src->stride + c) * ch;
                int y = (13933 * (int)px[0] + 46871 * (int)px[1] + 4732 * (int)px[2] + 32768) >> 16;
                y = y < 0 ? 0 : (y > 255 ? 255 : y);
                v = (float)y;
            } else {
                return ZO_ERR_UNSUPPORTED;
            }
            gray[(size_t)r * cols + c] = v;
        }
    zo_image g{gray.data(), rows, cols, cols}, ix{gx.data(), rows, cols, cols}, iy{gy.data(), rows, cols, cols};
    static const float sobel_x[9] = {-1, 0, 1, -2, 0, 2, -1, 0, 1};     // edges.zig:14-18
    static const float sobel_y[9] = {-1, -2, -1, 0, 0, 0, 1, 2, 1};     // :21-25
    int rc = zo::convolve(&g, &ix, ZO_PIX_F32, sobel_x, 3, 3, ZO_BORDER_REPLICATE);
    if (rc) return rc;
    if ((rc = zo::convolve(&g, &iy, ZO_PIX_F32, sobel_y, 3, 3, ZO_BORDER_REPLICATE))) return rc;
    for (uint32_t r = 0; r < rows; ++r)
        for (uint32_t c = 0; c < cols; ++c) {
            const float a = gx[(size_t)r * cols + c], b = gy[(size_t)r * cols + c];
            const float magnitude = std::sqrt(a * a + b * b);
            const float scaled = magnitude / 4.0f;
            const float cl = std::fmax(0.0f, std::fmin(255.0f, scaled));
            ((uint8_t*)dst->data)[(size_t)r * dst->stride + c] = (uint8_t)std::trunc(cl);
        }
    return ZO_OK;
}

// edges.zig:212-274 Edges(T).canny: luma -> f32, Gaussian (radius ceil(3 sigma), .replicate, :663-687), Sobel gx / gy with .replicate,
// magnitude sqrt(gx^2 + gy^2), direction-quantised non-maximum suppression (:691-763, borders stay 0), double threshold and
// breadth-first hysteresis over the 8-neighbourhood (:499-575).  dst is a binary (0 / 255) Image(u8).
int zo_canny(const zo_image* src, zo_image* dst, int pixfmt, float sigma, float low_threshold, float high_threshold) {
    if (!std::isfinite(sigma) || !std::isfinite(low_threshold) || !std::isfinite(high_threshold)) return ZO_ERR_INVALID_ARGUMENT;  // :221
    if (sigma < 0) return ZO_ERR_INVALID_SIGMA;                                                  // :224
    if (low_threshold < 0 || high_threshold < 0) return ZO_ERR_INVALID_THRESHOLD;                // :225
    if (low_threshold >= high_threshold) return ZO_ERR_INVALID_THRESHOLD;                        // :226
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;
    const uint32_t rows = src->rows, cols = src->cols;
    const size_t n = (size_t)rows * cols;
    std::vector<float> gray(n), blurred(n), gx(n), gy(n), mag(n);
    for (uint32_t r = 0; r < rows; ++r)                                                          // :229-236 as(f32, convertColor(u8, px))
        for (uint32_t c = 0; c < cols; ++c) {
            float v;
            if (pixfmt == ZO_PIX_F32) {                                                          // color.zig:114-118 float -> u8 through f64
                double d = (double)((const float*)src->data)[(size_t)r * src->stride + c];
                d = zo::zig_max(0.0, zo::zig_min(d, 1.0));   // std.math.clamp: NaN -> 1
                v = (float)(uint8_t)std::round(d * 255.0);
            } else if (pixfmt == ZO_PIX_U8) {
                v = (float)((const uint8_t*)src->data)[(size_t)r * src->stride + c];
            } else if (pixfmt == ZO_PIX_RGB8 || pixfmt == ZO_PIX_RGBA8) {
                const int ch = pixfmt == ZO_PIX_RGB8 ? 3 : 4;
                const uint8_t* px = (const uint8_t*)src->data + ((size_t)r * src->stride + c) * ch;
                int y = (13933 * (int)px[0] + 46871 * (int)px[1] + 4732 * (int)px[2] + 32768) >> 16;   // color.zig:1031-1041
                y = y < 0 ? 0 : (y > 255 ? 255 : y);
                v = (float)y;
            } else {
                return ZO_ERR_UNSUPPORTED;
            }
            gray[(size_t)r * cols + c] = v;
        }
    zo_image g{gray.data(), rows, cols, cols}, b{blurred.data(), rows, cols, cols}, ix{gx.data(), rows, cols, cols},
        iy{gy.data(), rows, cols, cols};
    int rc;
    if (sigma == 0) {                                                                            // :241-242
        blurred = gray;
    } else {                                                                                     // :663-687 (same taps as gaussianBlur)
        const size_t radius = (size_t)std::ceil(3.0f * sigma);
        std::vector<float> taps(2 * radius + 1);
        zo::gaussian_taps(sigma, taps.data(), (int)taps.size());
        if ((rc = zo::conv_separable(&g, &b, ZO_PIX_F32, taps.data(), (int)taps.size(), taps.data(), (int)taps.size(), ZO_BORDER_REPLICATE)))
            return rc;
    }
    static const float sobel_x[9] = {-1, 0, 1, -2, 0, 2, -1, 0, 1};     // edges.zig:14-18
    static const float sobel_y[9] = {-1, -2, -1, 0, 0, 0, 1, 2, 1};     // :21-25
    if ((rc = zo::convolve(&b, &ix, ZO_PIX_F32, sobel_x, 3, 3, ZO_BORDER_REPLICATE))) return rc;   // :253
    if ((rc = zo::convolve(&b, &iy, ZO_PIX_F32, sobel_y, 3, 3, ZO_BORDER_REPLICATE))) return rc;   // :254
    for (size_t i = 0; i < n; ++i) mag[i] = std::sqrt(gx[i] * gx[i] + gy[i] * gy[i]);              // :259-265

    std::vector<uint8_t> nms(n, 0);                                                              // :691-763
    const float K = 0.414213562f;
    if (rows >= 3 && cols >= 3) {
        for (uint32_t r = 1; r + 1 < rows; ++r)
            for (uint32_t c = 1; c + 1 < cols; ++c) {
                const float vx = gx[(size_t)r * cols + c], vy = gy[(size_t)r * cols + c];
                const float ax = std::fabs(vx), ay = std::fabs(vy);
                int dr1, dc1, dr2, dc2;
                if (ay <= K * ax) { dr1 = 0; dc1 = -1; dr2 = 0; dc2 = 1; }
                else if (ax <= K * ay) { dr1 = -1; dc1 = 0; dr2 = 1; dc2 = 0; }
                else if (vx * vy > 0) { dr1 = -1; dc1 = 1; dr2 = 1; dc2 = -1; }
                else { dr1 = -1; dc1 = -1; dr2 = 1; dc2 = 1; }
                const float m = mag[(size_t)r * cols + c];
                const float n1 = mag[(size_t)((int)r + dr1) * cols + (size_t)((int)c + dc1)];
                const float n2 = mag[(size_t)((int)r + dr2) * cols + (size_t)((int)c + dc2)];
                if (m >= n1 && m >= n2) nms[(size_t)r * cols + c] = 255;
            }
    }

    uint8_t* out = (uint8_t*)dst->data;                                                          // :499-575
    for (uint32_t r = 0; r < rows; ++r) std::memset(out + (size_t)r * dst->stride, 0, cols);
    std::vector<uint32_t> queue;
    queue.reserve(n);
    for (uint32_t r = 0; r < rows; ++r)
        for (uint32_t c = 0; c < cols; ++c)
            if (nms[(size_t)r * cols + c] > 0 && mag[(size_t)r * cols + c] >= high_threshold) {
                out[(size_t)r * dst->stride + c] = 255;
                queue.push_back(r * cols + c);
            }
    for (size_t pop = 0; pop < queue.size(); ++pop) {
        const uint32_t r = queue[pop] / cols, c = queue[pop] % cols;
        const uint32_t r0 = r > 0 ? r - 1 : 0, r1 = std::min(r + 2, rows), c0 = c > 0 ? c - 1 : 0, c1 = std::min(c + 2, cols);
        for (uint32_t nr = r0; nr < r1; ++nr)
            for (uint32_t nc = c0; nc < c1; ++nc) {
                if (nr == r && nc == c) continue;
                if (out[(size_t)nr * dst->stride + nc] > 0) continue;
                if (nms[(size_t)nr * cols + nc] > 0 && mag[(size_t)nr * cols + nc] >= low_threshold) {
                    out[(size_t)nr * dst->stride + nc] = 255;
                    queue.push_back(nr * cols + nc);
                }
            }
    }
    return ZO_OK;
}

int zo_gaussian_blur(const zo_image* src, zo_image* dst, int pixfmt, float sigma) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;  // image.zig:962
    if (sigma == 0) { zo::copy_image(src, dst, pixfmt); return ZO_OK; }                       // :966
    if (sigma < 0) return ZO_ERR_INVALID_SIGMA;                                               // :970
    const size_t radius = (size_t)std::ceil(3.0f * sigma);
    std::vector<float> taps(2 * radius + 1);
    zo::gaussian_taps(sigma, taps.data(), (int)taps.size());
    return zo::conv_separable(src, dst, pixfmt, taps.data(), (int)taps.size(), taps.data(), (int)taps.size(),
                              ZO_BORDER_MIRROR);  // :993
}

}  // extern "C"
