/*
 * zignal_b200.h -- C ABI of libzignal_b200.so: the H100 (sm_90a) implementation of zignal's
 * per-pixel image hot path.  This is the drop-in boundary: plain pointers and sizes, no C++ or
 * torch types.  A host shim in the reference's language (zig/zignal_b200.zig; C++ mirror in
 * zignal_b200/host/zignal.hpp; Python ctypes mirror in zignal_b200/) maps zignal's own
 * Image(T)/Matrix(T) method signatures onto these entry points (see INTEGRATION.md).
 *
 * The reference has no FFI on this path (callers invoke monomorphised Zig generics), so each entry
 * point cites the reference *method* it replaces, file:line under arrufat/zignal src/.
 *
 * Conventions
 *  - zb_image mirrors Image(T) (image.zig:97-102): row-major, `stride` in PIXELS, views allowed.
 *  - `pixfmt` replaces the comptime pixel type T.
 *  - zb_* image ops take DEVICE pointers and enqueue on `stream` (a cudaStream_t, NULL = default
 *    stream); they return after enqueueing.  zb_host_* twins take HOST pointers, stage through the
 *    library's device scratch and return when the result is back in host memory (the literal drop-in
 *    for an `Image.data` that lives in host memory).
 *  - Every function returns a zb_status (0 = ok) named after the Zig error it maps to.
 *  - Index range: the kernels hold a row index, and a channel element's or byte's index within a row, in an int (offsets from
 *    an image's start are 64-bit).  So every image op below returns ZB_ERR_UNSUPPORTED, before any allocation or launch, for an
 *    image (source or destination) with 2^31 rows or more, or with a row of 2^31 bytes or more (cols x pixel bytes).  Calls that
 *    the reference completes without computing anything are still completed: equal shapes or formats that copy (resize, convert),
 *    radius, distance, strength, sigma or iterations 0 (copy), dither NONE / AUTO (no-op).  The host-pointer twins refuse before
 *    staging.  zb_build_palette's adaptive mode refuses too rather than fall back to a fixed palette.  Not limited:
 *    zb_upload / zb_download / zb_copy / zb_set_border_zero, the histogram family (zb_histogram, zb_autocontrast, zb_equalize,
 *    zb_threshold_otsu: 2^32 pixels, below), fdm, the JPEG codec (65,535 per side) and zb_hough_find_lines.  Images with fewer
 *    rows and narrower rows but more than 2^32 bytes in all are accepted by every op; tests/test_gpu_index_range.py lists which
 *    op runs on which such shape.
 *  - Transcendental inputs (Gaussian taps, cos/sin of a rotation angle, Lanczos LUT) are computed
 *    on the host and cross the boundary as data, so every consumer sees identical values.
 */
#ifndef ZIGNAL_B200_H
#define ZIGNAL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZB_VERSION_MAJOR 0
#define ZB_VERSION_MINOR 1

typedef void* zb_stream; /* cudaStream_t */

/* Image(T): image.zig:97-102.  data: device pointer (zb_*) or host pointer (zb_host_*). */
typedef struct zb_image {
    void*    data;
    uint32_t rows;
    uint32_t cols;
    uint64_t stride; /* in pixels; == cols when contiguous (image.zig:355) */
} zb_image;

/* comptime pixel type T -> runtime tag */
typedef enum zb_pixfmt {
    ZB_PIX_U8 = 0,      /* Image(u8)                                                         */
    ZB_PIX_F32 = 1,     /* Image(f32)                                                        */
    ZB_PIX_RGB8 = 2,    /* Image(Rgb(u8)):  3 bytes r,g,b          color.zig:286-290         */
    ZB_PIX_RGBA8 = 3,   /* Image(Rgba(u8)): packed r,g,b,a         color.zig:400-405         */
    ZB_PIX_RGBAF32 = 4  /* Image(Rgba(f32)): 16-byte packed struct; filters act per channel  */
} zb_pixfmt;

/* BorderMode: border.zig:10-19 */
typedef enum zb_border { ZB_BORDER_ZERO = 0, ZB_BORDER_REPLICATE = 1, ZB_BORDER_MIRROR = 2, ZB_BORDER_WRAP = 3 } zb_border;

/* Interpolation: interpolation.zig:53-68 (union tag order; mitchell carries b, c) */
typedef enum zb_interp {
    ZB_INTERP_NEAREST = 0, ZB_INTERP_BILINEAR = 1, ZB_INTERP_BICUBIC = 2,
    ZB_INTERP_CATMULL_ROM = 3, ZB_INTERP_MITCHELL = 4, ZB_INTERP_LANCZOS = 5
} zb_interp;

/* geometry/transforms.zig:10,118,197 */
typedef enum zb_xform { ZB_XFORM_SIMILARITY = 0, ZB_XFORM_AFFINE = 1, ZB_XFORM_PROJECTIVE = 2 } zb_xform;

/* svd.zig:6-17 */
typedef enum zb_svd_mode { ZB_SVD_NO_U = 0, ZB_SVD_SKINNY_U = 1, ZB_SVD_FULL_U = 2 } zb_svd_mode;

/* Zig error names (image.zig:637,970,531-536; Matrix.zig:52-62; fdm.zig:114,142-143; pca.zig) */
typedef enum zb_status {
    ZB_OK = 0,
    ZB_ERR_DIMENSION_MISMATCH = 1, /* error.DimensionMismatch */
    ZB_ERR_INVALID_SIGMA = 2,      /* error.InvalidSigma      */
    ZB_ERR_UNSUPPORTED = 3,        /* (compile error in Zig: type not supported by this op) */
    ZB_ERR_NOT_CONVERGED = 4,      /* error.NotConverged / error.SvdFailed */
    ZB_ERR_INVALID_ARGUMENT = 5,
    ZB_ERR_OUT_OF_MEMORY = 6,      /* error.OutOfMemory       */
    ZB_ERR_DEVICE_FAILURE = 7,     /* CUDA / NCCL failure (new: error.DeviceFailure) */
    ZB_ERR_INVALID_SCALE_FACTOR = 8, /* error.InvalidScaleFactor (image.zig:531) */
    ZB_ERR_INVALID_DIMENSIONS = 9, /* error.InvalidDimensions (image.zig:536) */
    ZB_ERR_NO_TARGET_SET = 10,     /* fdm.zig:142 */
    ZB_ERR_NO_SOURCE_SET = 11,     /* fdm.zig:143 */
    ZB_ERR_INSUFFICIENT_DATA = 12, /* pca.zig:114-115 NoVectors / InsufficientData */
    ZB_ERR_INVALID_COMPONENTS = 13, /* pca.zig:123 */
    ZB_ERR_INVALID_THRESHOLD = 14, /* error.InvalidThreshold (edges.zig:225-226) */
    ZB_ERR_INVALID_PERCENTILE = 15, /* error.InvalidPercentile (order_statistic_blur.zig:49) */
    ZB_ERR_INVALID_TRIM = 16,      /* error.InvalidTrim (order_statistic_blur.zig:161) */
    ZB_ERR_IMAGE_TOO_SMALL = 17,   /* error.ImageTooSmall (metrics.zig:61) */
    ZB_ERR_NOT_SQUARE = 18,        /* error.NotSquare (eigen.zig:36) */
    ZB_ERR_NOT_SYMMETRIC = 19,     /* error.NotSymmetric (eigen.zig:54) */
    ZB_ERR_NOT_FINITE = 20,        /* error.NotFinite (eigen.zig:49) */
    ZB_ERR_INVALID_CUTOFF = 21,    /* error.InvalidCutoff (enhancement.zig:17) */
    ZB_ERR_INVALID_RADIUS = 22,    /* error.InvalidRadius (binary.zig:93) */
    ZB_ERR_INVALID_KERNEL_SIZE = 23, /* error.InvalidKernelSize (binary.zig:23-25) */
    ZB_ERR_INVALID_B_PARAMETER = 24, /* error.InvalidBParameter (ShenCastan.zig:40) */
    ZB_ERR_WINDOW_SIZE_MUST_BE_ODD = 25, /* error.WindowSizeMustBeOdd (ShenCastan.zig:41) */
    ZB_ERR_WINDOW_SIZE_TOO_SMALL = 26, /* error.WindowSizeTooSmall (ShenCastan.zig:42) */
    ZB_ERR_OUT_OF_BOUNDS = 27,     /* error.OutOfBounds (flood_fill.zig:68-70) */
    ZB_ERR_NO_PALETTE_COLORS = 28, /* error.NoPaletteColors (quantize.zig:241-243) */
    ZB_ERR_INVALID_IMAGE_DIMENSIONS = 29, /* error.InvalidImageDimensions (codecs/jpeg.zig:309-311) */
    ZB_ERR_IMAGE_TOO_LARGE = 30,   /* error.ImageTooLarge (codecs/jpeg.zig:312-314); also every jpeg.DecodeLimits error */
    ZB_ERR_INVALID_JPEG = 31       /* every decoder error of codecs/jpeg.zig that means a malformed stream (JpegError :2160-2201) */
} zb_status;

/* ------------------------------------------------------------------------------------------------
 * Runtime: device, streams, memory.  These back the Zig `std.mem.Allocator` vtable of the shim
 * (Image(T).init(dev_alloc, ...) / deinit, image.zig:124-158) and the pinned-host allocator.
 * ---------------------------------------------------------------------------------------------- */
int         zb_version(void);                 /* major*1000 + minor */
const char* zb_status_name(int status);
const char* zb_last_error(void);              /* thread-local text of the last CUDA failure */
int zb_device_count(int* count);
int zb_set_device(int ordinal);
int zb_get_device(int* ordinal);
int zb_sm_count(int* count);
int zb_stream_create(zb_stream* out);
int zb_stream_destroy(zb_stream s);
int zb_stream_synchronize(zb_stream s);
int zb_malloc(void** out, size_t bytes, zb_stream s);      /* cudaMallocAsync (stream-ordered pool) */
int zb_free(void* p, zb_stream s);                         /* cudaFreeAsync */
int zb_malloc_host(void** out, size_t bytes);              /* pinned host memory */
int zb_free_host(void* p);
/* Image-shaped copies (row pitch honoured on both sides); direction from the pointer kinds. */
/* Image.setBorder(rect, zeroes(T))   image.zig:198-229: zero everything outside [l, r) x [t, b) (the rect is clipped to the
 * image; an empty intersection zeroes the whole image).  Four strided memsets on the stream. */
int zb_set_border_zero(zb_image* img, int pixfmt, uint32_t l, uint32_t t, uint32_t r, uint32_t b, zb_stream s);
int zb_upload(const zb_image* host_src, zb_image* dev_dst, int pixfmt, zb_stream s);
int zb_download(const zb_image* dev_src, zb_image* host_dst, int pixfmt, zb_stream s);
int zb_copy(const zb_image* dev_src, zb_image* dev_dst, int pixfmt, zb_stream s); /* Image.copy, image.zig:375-392 */
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
uint64_t zb_kernel_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Filters
 * ---------------------------------------------------------------------------------------------- */
/* Host helper, image.zig:972-990: radius = ceil(3 sigma); taps exp(-x^2/(2 sigma^2)) in f32,
 * normalised by a sequential f32 sum.  Returns the tap count in *n (0 for sigma == 0). */
int zb_gaussian_taps(float sigma, float* taps, int cap, int* n);

/* Image.convolveSeparable(out, allocator, kernel_x, kernel_y, border)   image.zig:935-951,
 * convolution.zig:313-438.  kx/ky are HOST arrays.  In-place (src->data == dst->data) is allowed. */
int zb_conv_separable(const zb_image* src, zb_image* dst, int pixfmt,
                      const float* kx, int nx, const float* ky, int ny, int border, zb_stream s);
/* Sharding extension (no reference counterpart; SURVEY 8(e)): the same operation restricted to the OUTPUT rows
 * [row_begin, row_end) of dst.  src is still the whole image, so border handling and every value are identical to
 * the full call.  A row-block owner convolves the rows that do not depend on its halo while the halo exchange is in
 * flight, then the few boundary rows.  row_end == 0 means "to the last row". */
int zb_conv_separable_rows(const zb_image* src, zb_image* dst, int pixfmt,
                           const float* kx, int nx, const float* ky, int ny, int border,
                           uint32_t row_begin, uint32_t row_end, zb_stream s);
/* Image.convolve(out, allocator, kernel, border)   image.zig:917-931, convolution.zig:198-301.
 * kernel: HOST kh*kw row-major f32 (the comptime 2-D array after `as(f32, .)`). */
int zb_convolve(const zb_image* src, zb_image* dst, int pixfmt,
                const float* kernel, int kh, int kw, int border, zb_stream s);
/* Image.gaussianBlur(out, allocator, sigma)   image.zig:954-994 (always .mirror). */
int zb_gaussian_blur(const zb_image* src, zb_image* dst, int pixfmt, float sigma, zb_stream s);
/* Image.boxBlur(out, allocator, radius)   image.zig:635-648, integral.zig:148-269. */
int zb_box_blur(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, zb_stream s);
/* Image.sharpen(out, allocator, radius)   image.zig:785-799, integral.zig:273-422. */
int zb_sharpen(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, zb_stream s);
/* Image.integral: one f32 summed-area plane of a scalar image (integral.zig:41-78). sat: device rows*cols f32. */
int zb_integral_plane(const zb_image* src, int pixfmt, float* sat, zb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Resampling and geometry
 * ---------------------------------------------------------------------------------------------- */
/* Image.resize(out, allocator, method)   image.zig:523-525, interpolation.zig:89-191. */
int zb_resize(const zb_image* src, zb_image* dst, int pixfmt, int method, float mitchell_b, float mitchell_c, zb_stream s);
/* Image.rotateBounds(angle)   image.zig:570, transforms.zig:112-149 (host math). */
int zb_rotate_bounds(uint32_t rows, uint32_t cols, float angle, uint32_t* out_rows, uint32_t* out_cols);
/* Image.rotateInto(out, angle, method, border)   image.zig:564, transforms.zig:163-212. */
int zb_rotate_into(const zb_image* src, zb_image* dst, int pixfmt, float angle,
                   int method, float mitchell_b, float mitchell_c, int border, zb_stream s);
/* Same, with cos(angle) / sin(angle) supplied by the caller (transforms.zig:190-191 computes them with
 * Zig's @cos/@sin; passing them as data makes every consumer use identical values).  `angle` still
 * selects the orthogonal fast paths (transforms.zig:165-187). */
int zb_rotate_into_cs(const zb_image* src, zb_image* dst, int pixfmt, float angle, float cos_a, float sin_a,
                      int method, float mitchell_b, float mitchell_c, int border, zb_stream s);
/* Batched rotateInto: n images of identical shape stored back to back (image i starts
 * i*image_pitch_px pixels after image 0).  Same arithmetic per image as zb_rotate_into_cs. */
int zb_rotate_into_batch(const zb_image* src0, uint64_t src_image_pitch_px, zb_image* dst0, uint64_t dst_image_pitch_px,
                         uint32_t n_images, int pixfmt, float angle, float cos_a, float sin_a,
                         int method, float mitchell_b, float mitchell_c, int border, zb_stream s);
/* Image.warp(out, transform, method)   image.zig:621, transforms.zig:522-531 with
 * {Similarity,Affine,Projective}Transform.project  geometry/transforms.zig:39,147,224.
 * m (HOST): similarity/affine {m00,m01,m10,m11,b0,b1}; projective 9 values row-major. */
int zb_warp(const zb_image* src, zb_image* dst, int pixfmt, int xform_kind, const float* m,
            int method, float mitchell_b, float mitchell_c, zb_stream s);

/* Image.sobel(out, allocator)   image.zig:999-1009, edges.zig:33-73: gradient magnitude of the luma into an Image(u8)
 * (src: U8, F32, RGB8 or RGBA8; dst is always an 8-bit gray image of the same shape). */
int zb_sobel(const zb_image* src, zb_image* dst_u8, int pixfmt, zb_stream s);
/* Image.canny(out, allocator, sigma, low_threshold, high_threshold)   image.zig:1041-1063, edges.zig:212-274: luma -> Gaussian
 * (.replicate) -> Sobel -> non-maximum suppression -> double threshold + hysteresis, all on the device; dst receives 0 / 255.
 * Non-finite parameter: ZB_ERR_INVALID_ARGUMENT (error.InvalidParameter); sigma < 0: ZB_ERR_INVALID_SIGMA; negative thresholds
 * or low >= high: ZB_ERR_INVALID_THRESHOLD.  The hysteresis iterates to a fixed point, so this call waits for the stream. */
int zb_canny(const zb_image* src, zb_image* dst_u8, int pixfmt, float sigma, float low_threshold, float high_threshold, zb_stream s);
/* Image.shenCastan(out, allocator, opts)   image.zig:1015-1027, edges.zig:83-198, options ShenCastan.zig: luma (as for canny) -> ISEF
 * smoothing along rows then columns (:283-350, a = 1 - smooth, separately rounded f32 recurrences) -> binary Laplacian (smoothed - gray >= 0)
 * -> zero crossings (:356-414; forward E / S / SE / SW neighbours, or the 4-neighbourhood when use_nms) -> adaptive gradient |mean1 - mean0|
 * over the clipped window_size box from three f32 summed-area tables (:417-495) -> t_high from the histogram of the candidates' rounded
 * gradients (:139-170: target = floor(f32(total) * high_ratio), t_high = f32(min(idx, 255)) with idx one past the bin that reached the
 * target; t_low = low_rel * t_high) -> optional non-maximum suppression along the smoothed image's central differences (:582-656) ->
 * 255 where edge && g >= t_high, grown 8-connected through edge && g >= t_low when hysteresis (:499-575).  No candidate at all: all zeros.
 * src: U8, F32, RGB8 or RGBA8 (RGBA F32: ZB_ERR_UNSUPPORTED, as for canny); dst receives 0 / 255 and may be a strided view; a U8 src may
 * alias dst.  Errors, all decided before any device work, in this order: ZB_ERR_INVALID_ARGUMENT (NULL), ZB_ERR_UNSUPPORTED (pixel type),
 * ZB_ERR_DIMENSION_MISMATCH, then ShenCastan.validate's order (ShenCastan.zig:39-45): ZB_ERR_INVALID_B_PARAMETER (smooth not in (0, 1),
 * NaN included), ZB_ERR_WINDOW_SIZE_MUST_BE_ODD, ZB_ERR_WINDOW_SIZE_TOO_SMALL (below 3), ZB_ERR_INVALID_THRESHOLD (high_ratio, then
 * low_rel, not in (0, 1)).  An empty image is ok.  The thresholds stay on the device: without hysteresis the call returns after
 * enqueueing; with hysteresis it iterates to a fixed point as canny does and waits for the stream. */
int zb_shen_castan(const zb_image* src, zb_image* dst_u8, int pixfmt, float smooth, uint64_t window_size, float high_ratio, float low_rel,
                   int hysteresis, int use_nms, zb_stream s);

/* Order-statistic filters   image.zig:650-790, image/order_statistic_blur.zig:22-197 on 8-bit images (U8, RGB8, RGBA8; every channel
 * independently, :199-229).  One entry point for the family:
 *   Image.percentileBlur(out, radius, percentile, border)   mode ZB_ORDER_PERCENTILE, param = percentile in [0, 1]
 *   Image.medianBlur(out, radius)                            = percentile 0.5 with ZB_BORDER_MIRROR (:22-29)
 *   Image.minBlur / maxBlur(out, radius, border)             = percentile 0.0 / 1.0 (:83-101)
 *   Image.midpointBlur(out, radius, border)                  mode ZB_ORDER_MIDPOINT (param ignored)
 *   Image.alphaTrimmedMeanBlur(out, radius, trim, border)    mode ZB_ORDER_ALPHA_TRIMMED, param = trim fraction in [0, 0.5)
 * radius 0 copies; src may alias dst.  Errors in the reference's order: DimensionMismatch, (empty image: ok), InvalidTrim, (radius 0:
 * copy), InvalidPercentile, Unsupported (pixel type; also a window that no longer fits one SM's shared memory: radius beyond ~100 for
 * Rgba, ~220 for gray). */
enum { ZB_ORDER_PERCENTILE = 0, ZB_ORDER_MIDPOINT = 1, ZB_ORDER_ALPHA_TRIMMED = 2 };
int zb_order_blur(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, int mode, double param, int border, zb_stream s);

/* Image.motionBlur(out, allocator, .{ .linear = .{ .angle, .distance } })   image/motion_blur.zig:65-250.  cos / sin of the angle cross the
 * ABI as data (like rotateInto).  distance 0 copies; |sin| < 0.001 or |cos| < 0.001 is the reference's convolveSeparable branch (uniform
 * kernel, .replicate: the fused / tile convolution kernels); any other angle is the per-pixel line integral of bilinear samples
 * (src must not alias dst there). */
int zb_motion_blur_linear(const zb_image* src, zb_image* dst, int pixfmt, float angle, float cos_a, float sin_a, uint32_t distance, zb_stream s);
/* Image.motionBlur(..., .{ .radial_zoom | .radial_spin = .{ .center_x, .center_y, .strength } })   motion_blur.zig:252-436; spin != 0 selects
 * radial_spin.  Zoom is bit-exact; spin evaluates atan2 / cos / sin per sample on the device (last-bit libm differences: 1e-5 relative,
 * at most one 8-bit step on isolated pixels; on the outermost pixel ring the reference's own bounds test sits within an ulp of the image
 * edge, so a sample may be kept by one libm and dropped by another). */
int zb_motion_blur_radial(const zb_image* src, zb_image* dst, int pixfmt, float center_x, float center_y, float strength, int spin, zb_stream s);

/* Histogram-based and binary operations on 8-bit images.  Counts are u32 as in the reference, so an image of 2^32 pixels or more
 * returns ZB_ERR_UNSUPPORTED instead of wrapped counts.  Pixel formats other than U8 / RGB8 / RGBA8 (other than U8 for the threshold
 * and morphology calls, which take no pixfmt) are a compile error in the reference: ZB_ERR_UNSUPPORTED here.
 *
 * Image.histogram()   image.zig:1161-1185: counts[c * 256 + v] = pixels whose channel c is v (U8: 1 x 256, RGB8: 3 x 256, RGBA8: 4 x 256,
 * alpha included); only the view's own pixels count.  counts is a HOST array, so the call waits for the stream. */
int zb_histogram(const zb_image* src, int pixfmt, uint32_t* counts, zb_stream s);
/* Image.autocontrast(cutoff)   image.zig:804, enhancement.zig:11-80, in place.  Errors: ZB_ERR_UNSUPPORTED (pixel type), then
 * ZB_ERR_INVALID_CUTOFF for cutoff < 0, cutoff >= 0.5 or NaN.  cutoff_pixels = trunc(f32(rows * cols) * cutoff) (f32, on the host);
 * per channel min / max from findCutoffMin / findCutoffMax (histogram.zig:123-162), remap round(f32(clamp(v) - min) / f32(range) * 255).
 * RGB channels are remapped; RGBA alpha is left untouched. */
int zb_autocontrast(zb_image* img, int pixfmt, float cutoff, zb_stream s);
/* Image.equalize()   image.zig:824, enhancement.zig:84-252, in place, every channel (RGBA alpha too):
 * lut[i] = cdf[i] >= cdf_min ? (cdf[i] - cdf_min) * 255 / (total - cdf_min) : 0, identity when total == cdf_min.
 * Deviation: the numerator is formed in 64 bits.  The reference's u32 product overflows once total - cdf_min > 16,843,009 (e.g. any
 * 8192 x 8192 image), where it traps or is undefined; below that both agree bit for bit. */
int zb_equalize(zb_image* img, int pixfmt, zb_stream s);
/* Image(u8).thresholdOtsu(out)   image.zig:845, binary.zig:38-84: dst = src > t ? 255 : 0 with Otsu's t (sequential f64 search over the
 * 256 bins, first maximum wins), *threshold (HOST) = t; waits for the stream.  ZB_ERR_DIMENSION_MISMATCH first; an empty image gives
 * t = 0 and leaves dst untouched.  src may alias dst. */
int zb_threshold_otsu(const zb_image* src, zb_image* dst, uint8_t* threshold, zb_stream s);
/* Image(u8).thresholdAdaptiveMean(out, radius, c)   image.zig:858, binary.zig:86-119: dst = f32(src) > fl(fl(S / area) - c) ? 255 : 0,
 * S the boxBlur window sum of the f32 summed-area table, area the clipped window.  Errors in the reference's order:
 * ZB_ERR_DIMENSION_MISMATCH, ZB_ERR_INVALID_RADIUS (radius 0), then an empty image is ok.  src may alias dst. */
int zb_threshold_adaptive_mean(const zb_image* src, zb_image* dst, uint32_t radius, float c, zb_stream s);
/* Image(u8).dilateBinary / erodeBinary / openBinary / closeBinary(out, kernel, iterations)   image.zig:870-914, binary.zig:121-280.
 * kernel: HOST kernel_rows x kernel_cols bytes, non-zero = on, applied unreflected at (kr - rows/2, kc - cols/2); input pixels are
 * on when non-zero; dst receives 0 / 255; outside the image counts as background.  Errors: ZB_ERR_INVALID_KERNEL_SIZE (a zero or
 * even dimension, checked by Kernel.init before the call), ZB_ERR_DIMENSION_MISMATCH; iterations 0 copies.  Kernels larger than
 * 63 x 63 return ZB_ERR_UNSUPPORTED.  src may alias dst. */
enum { ZB_MORPH_DILATE = 0, ZB_MORPH_ERODE = 1, ZB_MORPH_OPEN = 2, ZB_MORPH_CLOSE = 3 };
int zb_morph_binary(const zb_image* src, zb_image* dst, const uint8_t* kernel, uint32_t kernel_rows, uint32_t kernel_cols,
                    uint32_t iterations, int op, zb_stream s);

/* HoughTransform   image/hough.zig:10-257: line detection on a binary edge map.  A zb_hough holds size, even_size and device copies of
 * the two i32 tables (uploaded by the first zb_hough_compute, on the device current then).
 *
 * zb_hough_create   hough.zig:38-66 (init): cos_table / sin_table are HOST arrays of `size` entries (the tables of the caller's own
 * HoughTransform.init), or NULL for trunc(65536 cos(theta) / sqrt(2)) / trunc(65536 sin(theta) / sqrt(2)), theta = t pi / even_size, in
 * f64 libm.  size <= 1: ZB_ERR_INVALID_ARGUMENT.  size > 32768: ZB_ERR_UNSUPPORTED (the reference's i32 rho overflows above that size).
 *
 * zb_hough_compute   hough.zig:75-139: every non-zero pixel of edges_u8 inside box (l, t, r, b; r, b exclusive) intersected with the
 * image votes once per angle column t into acc_u32[rr][t], rr = ((rho >> 1) + (offset << 1)) >> 16, rho = x_val cos[t] + y_val sin[t]
 * (i32, arithmetic shifts), kept when 0 <= rr < size.  The accumulator is ADDED to, not overwritten.  Both images may be strided views.
 * Errors, decided before any device work: ZB_ERR_INVALID_ARGUMENT (NULL), ZB_ERR_DIMENSION_MISMATCH (a box or an accumulator that is not
 * size x size).  An empty intersection launches nothing.  Returns after enqueueing.
 *
 * zb_hough_find_lines   hough.zig:142-257: local maxima of the interior of a device accumulator of any shape (votes >= threshold, no
 * 8-neighbour strictly greater), sorted by (score desc, row asc, col asc), greedy non-maximum suppression, f32 line geometry clipped to
 * [0, size]^2 with the handle's size.  *n receives the number of lines the reference returns; the first min(*n, cap) are written to the
 * HOST array out (NMS is prefix-stable, so these are the reference's first lines).  Waits for the stream. */
typedef struct zb_hough zb_hough;
typedef struct zb_hough_line { float angle, radius; uint32_t score; float p1x, p1y, p2x, p2y; } zb_hough_line;  /* Line, hough.zig:13-25 */
int zb_hough_create(uint32_t size, const int32_t* cos_table, const int32_t* sin_table, zb_hough** out);
int zb_hough_destroy(zb_hough* h);
int zb_hough_compute(const zb_hough* h, const zb_image* edges_u8, uint32_t l, uint32_t t, uint32_t r, uint32_t b,
                     zb_image* acc_u32, zb_stream s);
int zb_hough_find_lines(const zb_hough* h, const zb_image* acc_u32, uint32_t threshold, float angle_nms, float radius_nms,
                        zb_hough_line* out, uint32_t cap, uint32_t* n, zb_stream s);

/* Image.floodFill(allocator, start_row, start_col, fill_value, options)   image.zig:831-840, image/flood_fill.zig:59-131.  In place on a
 * device image (views allowed; nothing outside the view is touched).  fill_value: HOST pointer to one pixel of `pixfmt`.  connectivity: 4 or
 * 8.  mode: ZB_FLOOD_SEED compares each candidate with the seed pixel, ZB_FLOOD_NEIGHBOR with the adjacent pixel it is reached from.
 * Distance as pixelDistance (:28-51) in f64: |a - b| for U8 / F32; for RGB8 / RGBA8 / RGBAF32 the square root of the sum of squared
 * channel differences (alpha included), each operation rounded separately; a pixel joins when distance <= threshold (NaN never does).
 * Bit-identical to the reference's fill: union-find labelling of the region on the device, no host round trip, 4 B / pixel of
 * stream-ordered scratch.  Errors, all decided before any device work: ZB_ERR_INVALID_ARGUMENT (NULL image or fill_value, connectivity
 * other than 4 / 8, unknown mode), ZB_ERR_UNSUPPORTED (unknown pixfmt), ZB_ERR_OUT_OF_BOUNDS (start_row >= rows or start_col >= cols,
 * which includes an empty image; the image is left untouched), ZB_ERR_UNSUPPORTED (rows * cols >= 2^32: labels are u32).  Returns after
 * enqueueing. */
enum { ZB_FLOOD_SEED = 0, ZB_FLOOD_NEIGHBOR = 1 };
int zb_flood_fill(zb_image* img, int pixfmt, uint32_t start_row, uint32_t start_col, const void* fill_value, double threshold,
                  int connectivity, int mode, zb_stream s);

/* Colour quantization and dithering (image/quantize.zig, image/dither.zig), bit-identical to the reference.  Palettes are HOST arrays of
 * packed r, g, b bytes; a LUT is a DEVICE array of 32768 bytes, lut[r5][g5][b5] with r5 = r >> 3 (and so on).  Argument errors are all
 * decided before any device work: NULL pointers, an unknown mode, n == 0 or n > 256 (the reference packs the index into 8 bits) ->
 * ZB_ERR_INVALID_ARGUMENT; an unknown pixfmt -> ZB_ERR_UNSUPPORTED.
 * Deviations from the reference:
 *  1. a LUT index >= n reads a zero-padded 256-entry palette (the reference indexes its palette slice out of bounds);
 *  2. Atkinson on a 1-row image takes the bounds-checked branch (the reference computes rows - 2 in usize at dither.zig:271, which
 *     traps in safe builds and writes out of bounds in ReleaseFast).
 *
 * medianCut(T, gpa, image, palette, max_colors)   quantize.zig:175-412: writes min(colours, max_colors, cap) entries or fewer and sets
 * *n.  The histogram (count and first raster index per 5-bit key) is built on the device over the view, after convertColor to Rgb(u8);
 * the colours are ordered by first touch and cut on the host exactly as the reference does (std.sort.heap included).  No colour
 * (empty image, max_colors == 0 or cap == 0) -> ZB_ERR_NO_PALETTE_COLORS; rows * cols >= 2^32 -> ZB_ERR_UNSUPPORTED (the reference's
 * counts are u32).  Waits for the stream. */
int zb_median_cut(const zb_image* src, int pixfmt, uint16_t max_colors, uint8_t* palette, uint32_t cap, uint32_t* n, zb_stream s);
/* buildPalette(T, gpa, image, mode, palette)   quantize.zig:476-527 (PaletteMode tag order).  palette: HOST 256 x 3.  The fixed modes
 * ignore src and do no device work; ZB_PALETTE_ADAPTIVE runs zb_median_cut with cap 256 and, as the reference does, falls back to the
 * fixed 6x7x6 palette (252 colours) on any of its errors except ZB_ERR_DEVICE_FAILURE, which is returned.  Adaptive waits for the
 * stream. */
enum { ZB_PALETTE_FIXED_6X7X6 = 0, ZB_PALETTE_FIXED_VGA16 = 1, ZB_PALETTE_FIXED_WEB216 = 2, ZB_PALETTE_ADAPTIVE = 3 };
int zb_build_palette(const zb_image* src, int pixfmt, int mode, uint16_t max_colors, uint8_t* palette, uint32_t* n, zb_stream s);
/* ColorLookupTable.init(palette)   quantize.zig:66-159: for every 5-bit key the palette index minimising dist << 8 | i (the smallest
 * index wins ties).  palette: HOST n x 3; lut: DEVICE, 32768 bytes.  Returns after enqueueing. */
int zb_color_lut(const uint8_t* palette, uint32_t n, uint8_t* lut, zb_stream s);
/* dither.apply(img, palette, lut, mode)   dither.zig:34-331, in place on a device Rgb(u8) image or view (nothing outside the view is
 * touched).  Mode tag order; NONE and AUTO do nothing, as in apply (the caller resolves AUTO).  ORDERED is elementwise (8x8 Bayer
 * offset by view coordinates); FLOYD_STEINBERG and ATKINSON run as a wavefront of 32-row bands, with 8 B per column and band plus a
 * counter per band of stream-ordered scratch.  pixfmt other than ZB_PIX_RGB8 -> ZB_ERR_UNSUPPORTED (the reference asserts T == u8 on
 * Rgb).  Returns after enqueueing. */
enum { ZB_DITHER_NONE = 0, ZB_DITHER_FLOYD_STEINBERG = 1, ZB_DITHER_ATKINSON = 2, ZB_DITHER_ORDERED = 3, ZB_DITHER_AUTO = 4 };
int zb_dither(zb_image* img, int pixfmt, const uint8_t* palette, uint32_t n, const uint8_t* lut, int mode, zb_stream s);
/* ColorLookupTable.lookup(convertColor(Rgb, px)) per pixel   quantize.zig:163-168 (the GIF encoder's index map, gif.zig:900 / :916):
 * dst_u8[r, c] = lut[key of src[r, c]].  Any pixfmt; views allowed.  dst_u8 not of src's shape -> ZB_ERR_DIMENSION_MISMATCH.  Returns
 * after enqueueing. */
int zb_palette_lookup(const zb_image* src, int pixfmt, const uint8_t* lut, zb_image* dst_u8, zb_stream s);

/* Image.convert(allocator, TargetType) / convertInto(TargetType, out)   image.zig:396-421: out[r, c] = convertColor(TargetType, self[r, c])
 * (color.zig:108-151) between any two of the five pixel formats (equal formats copy, :398).  Bit-identical to the reference: integer BT.709
 * luma for 8-bit colours, separately rounded f32 arithmetic for float ones, u8 <-> float components as v / 255 and
 * round(255 * clamp(v, 0, 1)). */
int zb_convert(const zb_image* src, int src_pixfmt, zb_image* dst, int dst_pixfmt, zb_stream s);

/* Image.psnr(other) / Image.ssim(other) / Image.meanPixelError(other)   image.zig:1105-1147, image/metrics.zig:10-165: f64 quality
 * metrics of two device images of the same pixel format (U8, F32, RGB8, RGBA8, RGBAF32); *out is a HOST double, so each call waits
 * for the stream.  8-bit psnr / meanPixelError reproduce the reference's value exactly (integer sums); float formats and ssim
 * associate the final f64 sum differently (relative difference ~1e-15).  ssim: images under 11x11 give ZB_ERR_IMAGE_TOO_SMALL. */
int zb_psnr(const zb_image* a, const zb_image* b, int pixfmt, double* out, zb_stream s);
int zb_ssim(const zb_image* a, const zb_image* b, int pixfmt, double* out, zb_stream s);
int zb_mean_pixel_error(const zb_image* a, const zb_image* b, int pixfmt, double* out, zb_stream s);

/* Per-pixel visualisation methods of Image(T), every pixel format, views allowed everywhere (bytes outside a view are never touched).
 * Argument errors, all decided before any device work: NULL pointer -> ZB_ERR_INVALID_ARGUMENT, unknown pixfmt -> ZB_ERR_UNSUPPORTED,
 * images of different shapes -> ZB_ERR_DIMENSION_MISMATCH.
 *
 * Image.diff(out, other, opts)   image.zig:1139, image/diff.zig:27-203: out = |a - b| per channel (as f32), scaled (u8: round half
 * away from zero and saturate, NaN -> 255; f32: the product) or binary (max / 0 when the pixel differs: any channel, alpha included,
 * above threshold); force_opaque writes alpha as max and leaves it out of the stats sample.  out may alias a or b.  stats (HOST, or
 * NULL) receives DiffResult (diff.zig:19-22): RunningStats(f64, .summary) of one sample per pixel (the written value for U8 / F32, the
 * largest written non-alpha channel of a colour pixel, starting from 0) and diff_count.  8-bit formats: n, diff_count, sum, min and
 * max are the reference's bits; mean and variance are the exactly rounded rationals (the reference's Welford chain may differ in the
 * last bits).  Float formats: Welford per thread, Chan's merge in a fixed order (a repeated call returns the same bits).  variance =
 * m2 / (n - 1), 0 for n <= 1; every field 0 for an empty image.  Waits for the stream only when stats is non-NULL. */
typedef struct zb_diff_stats {
    uint64_t n, diff_count;
    double sum, mean, variance, min, max;
} zb_diff_stats;
int zb_diff(const zb_image* a, const zb_image* b, zb_image* out, int pixfmt, float threshold, float scale,
            int binary, int force_opaque, zb_diff_stats* stats, zb_stream s);
/* Colormap tags in the reference's union order (image/colormaps.zig:21-31). */
enum { ZB_COLORMAP_JET = 0, ZB_COLORMAP_HEAT = 1, ZB_COLORMAP_TURBO = 2, ZB_COLORMAP_VIRIDIS = 3, ZB_COLORMAP_INFERNO = 4 };
/* The 256 x 3 table of jet / heat / turbo (colormaps.zig:92-190), evaluated on the host in f64.  Viridis and inferno are data tables in
 * the reference and come from the caller (zignal's colormaps.viridis(i, 0, 255) / inferno): ZB_ERR_UNSUPPORTED here; an unknown map or
 * a NULL lut768 -> ZB_ERR_INVALID_ARGUMENT. */
int zb_colormap_lut(int map, uint8_t* lut768);
/* Image.applyColormap(allocator, map)   image.zig:1190-1247, colormaps.zig:43-86: dst_rgb8[r, c] = lut768[round(255 t)], t =
 * normalize(v, min, max) (meta.zig:255-260: 0 when any operand is NaN or max <= min, else clamped to [0, 1]).  v = meta.as(f64, px)
 * for U8 / F32 (0-255 for u8) and convertColor(f64, px) for RGB8 / RGBA8 / RGBAF32 (the Gray luma as a unit value).  A bound with
 * has_* == 0 comes from the view's pixels (NaN ignored; [0, 1] for an empty image); then max <= min gives max = min + 1.  The range is
 * found and applied on the device: no host round trip, returns after enqueueing.  lut768: HOST 256 x 3 bytes. */
int zb_apply_colormap(const zb_image* src, int pixfmt, const uint8_t* lut768, int has_min, double min, int has_max, double max,
                      zb_image* dst_rgb8, zb_stream s);
/* Image.flipLeftRight / flipTopBottom   image.zig:480-488, transforms.zig:28-45: in place; the middle column / row of an odd width /
 * height stays.  Image.invert   image.zig:494-511, color.zig:328,441: 255 - v for u8 components, 1.0 - c for Rgba(f32) (no clamp),
 * alpha kept; F32 -> ZB_ERR_UNSUPPORTED (a compile error in the reference).  All three return after enqueueing. */
int zb_flip_left_right(zb_image* img, int pixfmt, zb_stream s);
int zb_flip_top_bottom(zb_image* img, int pixfmt, zb_stream s);
int zb_invert(zb_image* img, int pixfmt, zb_stream s);

/* Image.extract(out, rect, angle, method, border)   image.zig / transforms.zig:232-283: resample the rectangle (l, t, r, b in source
 * coordinates, rotated by `angle` CCW around its centre; cos/sin cross the ABI as data like rotateInto) into dst; an axis-aligned
 * rect of dst's own size takes the copyRect path (:465-518).  Image.crop(rect) (:216-222) is
 * zb_extract(rect, 0, cos 1, sin 0, NEAREST, ZERO) into a round(height) x round(width) image. */
int zb_extract(const zb_image* src, zb_image* dst, int pixfmt, float rect_l, float rect_t, float rect_r, float rect_b, float angle,
               float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, int border, zb_stream s);

/* Image.insert(source, rect, angle, method, .none)   transforms.zig:293-376, the complement of extract: `source` (same pixel type as
 * `self`) is resampled into the rotated rectangle of `self`; pixels outside the rectangle are not touched.  (Blend modes:
 * zb_insert_blend; a source of another pixel type: zb_insert_from.) */
int zb_insert(zb_image* self, const zb_image* source, int pixfmt, float rect_l, float rect_t, float rect_r, float rect_b, float angle,
              float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, zb_stream s);
/* Image.insert(source, rect, angle, method, blend_mode) with a Blending mode (blending.zig:8-22, enum order): Rgba(u8) samples are
 * composited onto the Rgba(u8) destination by blendColors(u8, dest, sample, mode) (blending.zig:26-156, f32 arithmetic, Porter-Duff
 * "over" for the alpha); for every other pixel type the sample is assigned, as image.zig:67-95 assignPixel does. */
enum { ZB_BLEND_NONE = 0, ZB_BLEND_NORMAL, ZB_BLEND_MULTIPLY, ZB_BLEND_SCREEN, ZB_BLEND_OVERLAY, ZB_BLEND_SOFT_LIGHT, ZB_BLEND_HARD_LIGHT,
       ZB_BLEND_COLOR_DODGE, ZB_BLEND_COLOR_BURN, ZB_BLEND_DARKEN, ZB_BLEND_LIGHTEN, ZB_BLEND_DIFFERENCE, ZB_BLEND_EXCLUSION };
int zb_insert_blend(zb_image* self, const zb_image* source, int pixfmt, float rect_l, float rect_t, float rect_r, float rect_b, float angle,
                    float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, int blend_mode, zb_stream s);
/* Image.insert(source: anytype, ...) with a source of ANOTHER pixel type (transforms.zig:293, image.zig:67-95): samples are taken in the
 * source's type and converted per pixel with convertColor(DestType, sample); an Rgba(u8) source with a blend mode composites through
 * Rgba(u8): dest = convertColor(DestType, blend(convertColor(Rgba, dest), sample)).  Equal pixel types forward to zb_insert_blend. */
int zb_insert_from(zb_image* self, int self_pixfmt, const zb_image* source, int source_pixfmt, float rect_l, float rect_t, float rect_r,
                   float rect_b, float angle, float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, int blend_mode,
                   zb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Codecs
 * ---------------------------------------------------------------------------------------------- */
/* jpeg.Subsampling (codecs/jpeg.zig:262-282), enum order. */
typedef enum zb_jpeg_subsampling { ZB_JPEG_YUV444 = 0, ZB_JPEG_YUV422 = 1, ZB_JPEG_YUV420 = 2 } zb_jpeg_subsampling;
/* jpeg.EncodeOptions (codecs/jpeg.zig:284-290); zignal's defaults are quality 90, YUV420, 72 dpi, no comment (jpeg.save always uses
 * them).  comment: HOST bytes, NULL for no COM segment (a non-NULL comment of length 0 writes an empty COM). */
typedef struct zb_jpeg_options {
    uint8_t        quality;       /* clamped to [1, 100] (:464-465) */
    uint8_t        subsampling;   /* zb_jpeg_subsampling; ignored for ZB_PIX_U8 */
    uint16_t       density_dpi;
    const uint8_t* comment;
    uint32_t       comment_len;
} zb_jpeg_options;
/* A capacity that always suffices for zb_jpeg_encode: every block at its longest (the 11-bit DC code of category 11 with its
 * magnitude bits, then 63 AC symbols of a 16-bit code and 10 magnitude bits), whole bytes per block, doubled for 0xFF stuffing, plus
 * the header and EOI.  Same argument checks as zb_jpeg_encode; no device work. */
int zb_jpeg_encode_bound(uint32_t rows, uint32_t cols, int pixfmt, const zb_jpeg_options* opts, uint64_t* bytes);
/* jpeg.encode(T, allocator, image, options)   codecs/jpeg.zig:307-325 (encodeGrayscale :977-1042 for ZB_PIX_U8, encodeRgb :929-975
 * for ZB_PIX_RGB8, image.convert(Rgb) then encodeRgb for the other three formats): baseline JPEG (SOF0, 8-bit, the standard Huffman
 * tables), byte-identical to the reference.  src: DEVICE image, any pixel format, views allowed (the reference takes a contiguous
 * image).  Colour conversion, chroma averaging, FDCT, quantisation and the whole entropy-coded segment are computed on the device; the
 * header is written on the host.  *len receives the exact file size; the bytes go to out_host (HOST, cap bytes).  When cap < *len:
 * ZB_ERR_OUT_OF_MEMORY, nothing is written and *len still holds the size.  Errors, all decided before any device work:
 * ZB_ERR_INVALID_ARGUMENT (NULL src / opts / len, NULL out_host with cap > 0), ZB_ERR_UNSUPPORTED (unknown pixfmt),
 * ZB_ERR_INVALID_IMAGE_DIMENSIONS (rows or cols 0), ZB_ERR_IMAGE_TOO_LARGE (rows or cols above 65535), ZB_ERR_INVALID_ARGUMENT
 * (subsampling > 2, or a comment longer than 65533 bytes, whose segment length would not fit its u16).  Scratch that cannot be
 * allocated: ZB_ERR_OUT_OF_MEMORY.  Waits for the stream. */
int zb_jpeg_encode(const zb_image* src, int pixfmt, const zb_jpeg_options* opts, uint8_t* out_host, uint64_t cap, uint64_t* len,
                   zb_stream s);
/* jpeg.DecodeLimits (codecs/jpeg.zig:19-33); 0 disables a limit.  A NULL limits pointer means the reference's defaults:
 * 100 MiB, 100 MiB, 8192, 8192, 67108864 pixels, 1048576 blocks, 64 scans. */
typedef struct zb_jpeg_limits {
    uint64_t max_jpeg_bytes;
    uint64_t max_marker_bytes;
    uint32_t max_width;
    uint32_t max_height;
    uint64_t max_pixels;
    uint64_t max_blocks;
    uint64_t max_scans;
} zb_jpeg_limits;
/* jpeg.Header (codecs/jpeg.zig:61-73) as getInfo returns it. */
typedef struct zb_jpeg_header {
    uint32_t width;
    uint32_t height;
    int32_t  progressive;      /* frame_type: 0 baseline, 1 progressive (SOF2) */
    int32_t  num_components;
    int32_t  precision;
    int32_t  subsampling;      /* zb_jpeg_subsampling, or -1 for null (grayscale or another layout) */
} zb_jpeg_header;
/* jpeg.getInfo(reader, limits)   codecs/jpeg.zig:77-180, over the HOST bytes data[0, len): the first SOF's header, progressive
 * files included.  Host only.  Errors: ZB_ERR_IMAGE_TOO_LARGE (a max_jpeg_bytes or marker-count limit), ZB_ERR_INVALID_JPEG (no SOI,
 * EOI before any SOF, a marker length below 2, an SOF shorter than 6 bytes, or the end of the data). */
int zb_jpeg_info(const uint8_t* data, uint64_t len, const zb_jpeg_limits* limits, zb_jpeg_header* out);
/* jpeg.loadFromBytes(T, allocator, data, limits)   codecs/jpeg.zig:2825-2851 for baseline streams: decode (:2035-2157) ->
 * toNativeImage (:2786-2820) -> image.convert(T), pixel for pixel equal to the reference.  data: HOST bytes (one host-to-device copy
 * of the bytes after the SOS header; the host parses only the segments before it).  dst: DEVICE image of any pixel format, views
 * allowed, with exactly the frame's rows (height) and cols (width), else ZB_ERR_DIMENSION_MISMATCH.  Accepted: SOF0, 8-bit, one
 * component, or three at 4:4:4, 4:2:2, 4:2:0 or 4:1:1; any DHT / DQT the reference parses (16-bit tables included); DRI restart
 * intervals; truncated scans (what was decoded is kept, every later block is zero).  Only the first scan is decoded, as in the
 * reference.  Entropy decoding, IDCT and colour conversion all run on the device (DESIGN.md §4.9).
 * Deliberate differences from the reference (DESIGN.md §7): restart interval i starts at the byte after the i-th RST marker (T.81
 * F.2.2.5; a missing marker ends the decode as a truncation does), and i32 overflow on adversarial streams wraps.
 * Status mapping, all but the last decided before any device work:
 *   ZB_ERR_UNSUPPORTED: SOF2 (progressive; the reference decodes it, this port does not), and every error.Unsupported* of the
 *     reference (SOF1, SOF3, DAC, DHP, DNL, 12 / 16-bit or other precision, 4 components, sampling factors above 4, other layouts),
 *     and an unknown pixfmt;
 *   ZB_ERR_IMAGE_TOO_LARGE: ImageTooLarge, JpegDataTooLarge, MarkerDataLimitExceeded, BlockMemoryLimitExceeded;
 *   ZB_ERR_INVALID_JPEG: every other reference error (InvalidJpegFile, InvalidMarker, InvalidSOF, DuplicateSOF, InvalidDHT,
 *     InvalidDQT, InvalidSOS, InvalidDRI, InvalidComponentCount, InvalidHuffmanTable, NoScanData, UnexpectedEndOfData outside the
 *     scan, MissingQuantTable, BlockStorageNotAllocated), a scan component id that names no frame component, or one named twice;
 *   ZB_ERR_INVALID_JPEG after the device decode: InvalidHuffmanCode, InvalidDCCoefficient, InvalidACCoefficient or
 *     MissingHuffmanTable met before the data ran out (the image is then undefined);
 *   ZB_ERR_INVALID_ARGUMENT (NULL dst, NULL data with len > 0, NULL dst data, stride < cols), ZB_ERR_OUT_OF_MEMORY (scratch).
 * Waits for the stream. */
int zb_jpeg_decode(const uint8_t* data, uint64_t len, const zb_jpeg_limits* limits, zb_image* dst, int pixfmt, zb_stream s);
/* jpeg.loadFromBytes for n files in one call.  File i (HOST bytes data[i][0, len[i])) is decoded into the DEVICE image dst[i] as
 * pixfmt[i]; status[i] receives exactly what zb_jpeg_decode(data[i], len[i], limits, &dst[i], pixfmt[i], s) would return, and when
 * it is ZB_OK dst[i] holds exactly that call's pixels.  limits applies to each file separately.  Files refused on the host (header
 * and limit errors, a wrong destination shape or pixel format, a NULL destination, Unsupported) leave their image untouched; a file
 * that fails on the device (ZB_ERR_INVALID_JPEG) leaves it undefined.  Destination images must not overlap each other.
 * The files' scans go to the device in one copy and every stage runs once for the whole batch, so the host waits the same number
 * of times for one file as for many (DESIGN.md §4.9).
 * Returns ZB_OK once every file has been attempted (n = 0: no device work), ZB_ERR_INVALID_ARGUMENT for a NULL array with n > 0,
 * ZB_ERR_OUT_OF_MEMORY when the call's scratch cannot be allocated (the statuses are then undefined).  Waits for the stream. */
int zb_jpeg_decode_batch(uint32_t n, const uint8_t* const* data, const uint64_t* len, const zb_jpeg_limits* limits, zb_image* dst,
                         const int* pixfmt, int* status, zb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Linear algebra behind fdm / pca
 * ---------------------------------------------------------------------------------------------- */
/* Matrix.gemm(trans_a, other, trans_b, alpha, beta, c)   Matrix.zig:696-822.
 * All matrices DEVICE, row-major, contiguous.  c may be NULL.  out is a_rows x b_cols. */
int zb_gemm_f32(const float* a, uint32_t a_rows, uint32_t a_cols, int trans_a,
                const float* b, uint32_t b_rows, uint32_t b_cols, int trans_b,
                float alpha, float beta, const float* c, float* out, zb_stream s);
int zb_gemm_f64(const double* a, uint32_t a_rows, uint32_t a_cols, int trans_a,
                const double* b, uint32_t b_rows, uint32_t b_cols, int trans_b,
                double alpha, double beta, const double* c, double* out, zb_stream s);
/* Pca.fit's centering step (pca.zig:135-154): mean[j] = sum_i x[i][j] / n (when compute_mean != 0; f64 accumulation),
 * centered = x - mean (skipped when NULL).  Pca.transform (pca.zig:300-308) calls it with compute_mean = 0.  DEVICE pointers. */
int zb_center_columns_f32(const float* x, uint32_t n, uint32_t dim, float* mean, int compute_mean, float* centered, zb_stream s);
int zb_center_columns_f64(const double* x, uint32_t n, uint32_t dim, double* mean, int compute_mean, double* centered, zb_stream s);
/* Matrix.svd / SMatrix.svd   Matrix.zig:1570, SMatrix.zig:804, svd.zig:80-496.  HOST matrices.
 * a: m x n row-major, m >= n.  u: m x (mode==FULL ? m : n) or NULL; s: n (descending); v: n x n or NULL.
 * *converged receives 0 or a non-zero failure mark (svd.zig:79).
 * Computed by a one-sided Jacobi method with a parallel pair ordering on the GPU (n >= 24; smaller matrices run the same
 * algorithm on the host), not by the reference's sequential Golub-Reinsch: singular values agree to sqrt(eps) (to high relative
 * accuracy, in fact), U and V are orthonormal and reconstruct A, but the SIGN of each (u_i, v_i) pair and the basis inside a
 * cluster of equal singular values are the decomposition's usual freedom and may differ from the reference's. */
int zb_svd_f64(const double* a, uint32_t m, uint32_t n, int mode, int with_v, double* u, double* s, double* v, uint64_t* converged);
int zb_svd_f32(const float* a, uint32_t m, uint32_t n, int mode, int with_v, float* u, float* s, float* v, uint64_t* converged);
/* The same decomposition for a matrix that already lives on the device (Pca.fit: the covariance from zb_gemm never leaves the
 * GPU, pca.zig:331-425).  d_a: m x n row-major DEVICE (not modified); d_u: m x n skinny U or NULL; d_s: n; d_v: n x n or NULL --
 * all DEVICE.  Returns after the stream has finished. */
int zb_svd_dev_f64(const double* d_a, uint32_t m, uint32_t n, double* d_u, double* d_s, double* d_v, uint64_t* converged, zb_stream s);
int zb_svd_dev_f32(const float* d_a, uint32_t m, uint32_t n, float* d_u, float* d_s, float* d_v, uint64_t* converged, zb_stream s);
/* Matrix.eigh(allocator)   matrix/eigen.zig:34-136: symmetric eigendecomposition (HOST pointers, row-major n x n).  values[n] ascending,
 * vectors[n * n] with the matching unit eigenvectors as columns.  ZB_ERR_NOT_SQUARE, ZB_ERR_NOT_FINITE (NaN / inf entry),
 * ZB_ERR_NOT_SYMMETRIC (|a_ij - a_ji| > max|a| * sqrt(eps)), in the reference's order.  Two-sided Jacobi with a parallel pair
 * ordering on the GPU (n >= 24, host below): same eigenvalues to eps * |A|, eigenvectors up to sign. */
int zb_eigh_f64(const double* a, uint32_t rows, uint32_t cols, double* values, double* vectors);
int zb_eigh_f32(const float* a, uint32_t rows, uint32_t cols, float* values, float* vectors);

/* ------------------------------------------------------------------------------------------------
 * Feature distribution matching   fdm.zig:19-275
 * ---------------------------------------------------------------------------------------------- */
typedef struct zb_fdm zb_fdm;                       /* FeatureDistributionMatching(T) state, fdm.zig:22-39 */
int zb_fdm_create(zb_fdm** out, int pixfmt);        /* .init   fdm.zig:42 ; pixfmt in {U8, RGB8, RGBA8} (fdm.zig:20) */
int zb_fdm_destroy(zb_fdm* f);                      /* .deinit fdm.zig:61 */
int zb_fdm_set_target(zb_fdm* f, const zb_image* target, zb_stream s);  /* fdm.zig:68  (device image, contiguous) */
int zb_fdm_set_source(zb_fdm* f, zb_image* source);                      /* fdm.zig:127 */
int zb_fdm_update(zb_fdm* f, zb_stream s);                               /* fdm.zig:141 (in place on source) */
int zb_fdm_match(zb_fdm* f, zb_image* source, const zb_image* target, zb_stream s); /* fdm.zig:133 */
/* The statistics pass alone: exact integer moment sums of a u8 image (n, sum x_i, sum x_i x_j, is_gray)
 * -- the quantities one all-reduce combines across GPUs.  sums: HOST u64[11] =
 * {n, Sr, Sg, Sb, Srr, Srg, Srb, Sgg, Sgb, Sbb, non_gray_count}.  as_luma selects fdm.zig:157-162. */
int zb_fdm_moments(const zb_image* img, int pixfmt, int as_luma, uint64_t* sums11, zb_stream s);
/* Install externally reduced moments (multi-GPU: after the all-reduce) as target / source statistics. */
int zb_fdm_set_target_moments(zb_fdm* f, const uint64_t* sums11);
int zb_fdm_update_with_moments(zb_fdm* f, const uint64_t* source_sums11, zb_stream s);
/* zb_fdm_update queues its three kernels (moments, the 3x3 solve, the map) on the stream and returns; the solve's result
 * (0, or ZB_ERR_NOT_CONVERGED = error.SvdFailed, fdm.zig:216) stays on the device.  This call waits for the stream and
 * returns it. */
int zb_fdm_status(zb_fdm* f, zb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU: one process per GPU, a large image sharded into row blocks (SURVEY.md 8(e)).
 * The reference is single-process, so there is no reference counterpart: these entry points are what a
 * Zig host running one process per GPU binds to shard Image.convolveSeparable / gaussianBlur (image.zig:935-994),
 * any other neighbourhood filter, fdm.update (fdm.zig:141-273) and batches of rotate / resize.
 *
 * Plumbing: NCCL (dlopen'ed at run time) bootstraps the communicator and exchanges CUDA IPC handles; the data
 * path is NVLink peer memory.  The RGBA f32 convolution kernel copies the `half` edge rows of the row
 * neighbours from their memory into its own halo rows in a prologue -- one launch per step, no separate exchange
 * -- and carries the whole synchronisation in a pair of flags per neighbour (blocks need halo_cap >= 8 for this
 * kernel); every other filter uses zb_shard_halo_exchange (one pull
 * kernel over NVLink; NCCL send/recv when IPC mappings are unavailable) followed by its ordinary entry point
 * on the extended block.  All ranks must issue the same sequence of zb_shard_* calls (SPMD).
 * ---------------------------------------------------------------------------------------------- */
typedef struct zb_shard_comm zb_shard_comm;     /* one per process / GPU */
typedef struct zb_shard_image zb_shard_image;   /* a global image = `world` row blocks stacked in rank order */
#define ZB_SHARD_ID_BYTES 128
/* Rank 0 creates the id and hands it to the other ranks out of band (the host's own launcher); then every rank
 * creates its communicator on its current device.  world == 1 needs no id (and no NCCL). */
int zb_shard_unique_id(uint8_t* id128);
int zb_shard_comm_create(zb_shard_comm** out, int rank, int world, const uint8_t* id128);
int zb_shard_comm_destroy(zb_shard_comm* c);
int zb_shard_comm_info(const zb_shard_comm* c, int* rank, int* world, int* peer_access /* 1: IPC peer mappings in use */);
/* Waits for the stream; ZB_ERR_DEVICE_FAILURE if a kernel gave up waiting for a neighbour (a rank died or the ranks'
 * call sequences diverged) instead of hanging the GPU. */
int zb_shard_status(zb_shard_comm* c, zb_stream s);
/* Symmetric allocation (collective, same order and size on every rank): device memory every rank can address. */
int zb_shard_alloc(zb_shard_comm* c, size_t bytes, void** out);
int zb_shard_free(zb_shard_comm* c, void* p);
/* Describe this rank's row block (inside a zb_shard_alloc allocation, with `halo_cap` spare rows of the same stride above
 * and below it) of the global image (collective: the ranks learn each other's block heights and addresses). */
int zb_shard_image_create(zb_shard_comm* c, const zb_image* block, uint32_t halo_cap, int pixfmt, zb_shard_image** out);
int zb_shard_image_destroy(zb_shard_image* img);
int zb_shard_image_block(const zb_shard_image* img, zb_image* block);   /* this rank's block as a plain zb_image */
/* Contiguous share [lo, hi) of n_items for `rank` (batches of rotate / resize / warp: no exchange).  Pure host arithmetic. */
int zb_shard_split(uint32_t n_items, int rank, int world, uint32_t* lo, uint32_t* hi);
/* Fill the `reach` halo rows next to each row neighbour with the neighbour's edge rows (global edges are left to the filter's own
 * border mode; ZB_BORDER_WRAP closes the ring).  One kernel on `s`; when it completes, no neighbour is still reading this block. */
int zb_shard_halo_exchange(zb_shard_comm* c, zb_shard_image* img, uint32_t reach, int border, zb_stream s);
/* The block plus the halo rows that zb_shard_halo_exchange filled, as a zb_image for any zb_* filter; *interior_first = index of
 * the block's first row inside the view.  Rows of the result within `reach` of a neighbour-side end are halo rows (discard). */
int zb_shard_view(const zb_shard_image* img, uint32_t reach, int border, zb_image* view, uint32_t* interior_first);
/* Image.convolveSeparable / gaussianBlur of the GLOBAL image; src / dst: the same partition.  Bit-identical to the single-GPU
 * call on the whole image. */
int zb_shard_conv_separable(zb_shard_comm* c, const zb_shard_image* src, zb_shard_image* dst,
                            const float* kx, int nx, const float* ky, int ny, int border, zb_stream s);
int zb_shard_gaussian_blur(zb_shard_comm* c, const zb_shard_image* src, zb_shard_image* dst, float sigma, zb_stream s);
/* In-place sum over all ranks of a device buffer (dtype 0 = f32, 1 = f64, 2 = u64): PCA's partial X^T X products (pca.zig:338),
 * moment sums.  NCCL all-reduce. */
int zb_shard_allreduce(zb_shard_comm* c, void* dev_buf, size_t count, int dtype, zb_stream s);
/* fdm on a row-sharded image: every rank passes its block.  set_target: local moments + one all-reduce; update (zb_fdm_set_source
 * with the local block first): the statistics kernel all-gathers the 11 sums over NVLink peer memory in its last block, solves and
 * the map follows -- nothing leaves the device.  The result equals the single-GPU result on the whole image bit for bit. */
int zb_shard_fdm_set_target(zb_shard_comm* c, zb_fdm* f, const zb_image* target_block, zb_stream s);
int zb_shard_fdm_update(zb_shard_comm* c, zb_fdm* f, zb_stream s);
/* Testing aid: 0 = automatic, 1 = force the NCCL send/recv halo exchange, 2 = force the peer pull kernel for every format. */
int zb_shard_tune_path(int path);

/* ------------------------------------------------------------------------------------------------
 * Host-pointer twins (H2D + op + D2H inside the call; returns when dst is valid on the host).
 * ---------------------------------------------------------------------------------------------- */
int zb_host_conv_separable(const zb_image* src, zb_image* dst, int pixfmt,
                           const float* kx, int nx, const float* ky, int ny, int border);
int zb_host_convolve(const zb_image* src, zb_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border);
int zb_host_gaussian_blur(const zb_image* src, zb_image* dst, int pixfmt, float sigma);
int zb_host_box_blur(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius);
int zb_host_sharpen(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius);
int zb_host_resize(const zb_image* src, zb_image* dst, int pixfmt, int method, float mitchell_b, float mitchell_c);
int zb_host_rotate_into(const zb_image* src, zb_image* dst, int pixfmt, float angle, int method,
                        float mitchell_b, float mitchell_c, int border);
int zb_host_warp(const zb_image* src, zb_image* dst, int pixfmt, int xform_kind, const float* m,
                 int method, float mitchell_b, float mitchell_c);
int zb_host_fdm_match(zb_image* source, const zb_image* target, int pixfmt);

/* ------------------------------------------------------------------------------------------------
 * Tuning / introspection (not part of the drop-in surface)
 * ---------------------------------------------------------------------------------------------- */
/* Selects the arithmetic of the fused f32 separable kernel: 0 = FFMA (default, <= 1e-6 rel. from the
 * reference), 1 = unfused mul+add in the reference's order (bit-exact with it for finite data). */
int zb_set_exact_f32(int on);
/* Forces the generic (two-pass through HBM) separable path; used by tests to cross-check kernels. */
int zb_set_force_generic(int on);
/* Kernel tuning knobs for experiments ("conv.u8_fmath" 0|1,
 * "host.band_rows": rows per PCIe band of the pipelined host-pointer path, 0 = stage the whole image,
 * "conv.u8_dp" 0|1, "conv.edge_fast" 0|1 (x borders of .replicate / .mirror as in-stage copies), "sobel.tile" 0|1, "jacobi.cluster" 0|1 (SVD inside one cluster's shared memory when it fits), "rotate.tile" 0 gather kernel |
 * 1 shared-memory tile kernel where it applies). */
int zb_tune(const char* key, int value);
/* Name of the kernel variant the last zb_conv_separable call selected on this thread. */
const char* zb_last_kernel(void);
/* Jacobi sweeps the last zb_svd_* / zb_eigh_* call on this thread needed (60 = the limit: not converged). */
int zb_last_sweeps(void);

#ifdef __cplusplus
}
#endif
#endif /* ZIGNAL_B200_H */
