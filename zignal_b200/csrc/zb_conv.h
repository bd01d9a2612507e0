// zb_conv.h -- internal interface between the convolution translation units.
#pragma once
#include "zb_internal.h"

namespace zb {

constexpr int kMaxTaps = 1023;     // per separable axis (generic path)
constexpr int kMaxTaps2D = 1024;   // kh*kw (generic dense path)

// Band plan of the persistent (band x strip) convolution kernels, whose CTAs take units in band-major order: bands of about
// kBandTargetRows rows, then as many bands as fit in the same number of waves of `sm_count` units; band heights are a multiple
// of the kernels' 8-row chunk and at least 64 rows.
constexpr int kBandTargetRows = 256;
struct BandPlan {
    int n_bands, band_rows;
};
static inline BandPlan plan_bands(int nrows, int n_strips, int sm_count) {
    int n_bands = (nrows + kBandTargetRows - 1) / kBandTargetRows;
    const long long waves = ((long long)n_bands * n_strips + sm_count - 1) / sm_count;
    const int nb2 = (int)((waves * sm_count) / n_strips);
    if (nb2 > n_bands) n_bands = nb2;
    int band_rows = (nrows + n_bands - 1) / n_bands;
    band_rows = ((band_rows + 7) / 8) * 8;
    if (band_rows < 64) band_rows = 64;
    return {(nrows + band_rows - 1) / band_rows, band_rows};
}

// zb_conv_generic.cu
int conv_separable_generic(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny,
                           int border, cudaStream_t s);
int convolve_generic(const zb_image* src, zb_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border, cudaStream_t s);

// zb_conv_fused.cu: single-pass (read once, write once) separable convolution of interleaved RGBA f32.
// Returns ZB_ERR_UNSUPPORTED when the configuration is outside the fused kernel's envelope; the caller
// then uses the generic path.  [row0, row1) restricts the OUTPUT rows produced (row1 < 0: all) -- the host pipeline
// computes a band as soon as the rows it reads have been uploaded.
int conv_separable_fused_rgbaf32(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border,
                                 bool exact, cudaStream_t s, int row0 = 0, int row1 = -1);

// zb_conv_fused_u8.cu: single-pass separable convolution of interleaved Rgba(u8) (i32 accumulators, provably overflow-free taps).
int conv_separable_fused_rgba8(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border,
                               cudaStream_t s, int row0 = 0, int row1 = -1);

// zb_conv_tile_u8.cu: single-pass (shared-memory tile) separable convolution of any 8-bit format / alignment / border mode.
int conv_separable_tile_u8(const zb_image* src, zb_image* dst, int channels, const float* kx, int nx, const float* ky, int ny, int border,
                           cudaStream_t s);
// Dense kernels up to 7 x 7 on 8-bit images from shared-memory tiles (zb_conv_tile_u8.cu); ZB_ERR_UNSUPPORTED outside its envelope.
int convolve_tile_u8(const zb_image* src, zb_image* dst, int channels, const int32_t* ki, int kh, int kw, int border, cudaStream_t s);
// Image.sobel of an 8-bit image (gray / Rgb / Rgba) from shared-memory byte tiles (zb_conv_tile_u8.cu); ZB_ERR_UNSUPPORTED outside its envelope.
int sobel_tile_u8(const zb_image* src, zb_image* dst, int pixfmt, cudaStream_t s);

}  // namespace zb
