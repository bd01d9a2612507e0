// zb_warp.cu -- Image.rotateBounds / rotateInto / warp: inverse-mapped gather kernels.
// Reference: transforms.zig:112-149 (rotateBounds), :163-212 (rotateInto; fast paths within 1e-6 rad
// of k*pi/2 :165-187), :385-462 (rotate0/90/180/270 with centred placement and zeroed margins),
// :522-531 (warp, always .mirror), image.zig:322-327 (centre = (cols/2, rows/2) as f32),
// geometry/transforms.zig:39-42,147-150 (affine project: (m0*x + m1*y) + b, no fusion),
// :224-231 (projective: multiply by 1/w when w != 0).
// One thread per destination pixel; a CTA covers a 32x8 destination tile as 4x2 warps of 8x4 pixels, so that a
// warp's source footprint is a ~9x9 pixel patch (8-12 sectors per gather) for any rotation angle instead of a
// 32-pixel diagonal (one sector per lane).  Compiled with -fmad=false (coordinate math is the
// reference's unfused f32 sequence, which the u8 outputs depend on bit for bit).
#include <algorithm>
#include <cmath>
#include <mutex>

#include "zb_host_stage.h"
#include "zb_blend.cuh"
#include "zb_sample.cuh"
#include "zb_warp.h"

namespace zb {

namespace {

constexpr float TAU_F = 6.283185307179586f;
constexpr float PI_F = 3.141592653589793f;

// Zig's float @mod: a = frem(l, r); l < 0 ? frem(a + r, r) : a
static inline float zig_mod_f32(float l, float r) {
    const float a = std::fmod(l, r);
    return l < 0 ? std::fmod(a + r, r) : a;
}
// transforms.zig:114-136 / :165-187: 0 general, 1 = 0deg, 2 = 90, 3 = 180, 4 = 270
static int rotate_class(float angle) {
    const float n = zig_mod_f32(angle, TAU_F);
    const float eps = 1e-6f;
    if (std::fabs(n) < eps || std::fabs(n - TAU_F) < eps) return 1;
    if (std::fabs(n - PI_F / 2.0f) < eps) return 2;
    if (std::fabs(n - PI_F) < eps) return 3;
    if (std::fabs(n - 3.0f * PI_F / 2.0f) < eps) return 4;
    return 0;
}

// thread -> pixel of the CTA's 32x8 tile: warp w owns the 8x4 patch at (8 * (w & 3), 4 * (w >> 2))
__device__ __forceinline__ int patch_col(unsigned t) { return (int)(((t >> 5) & 3u) * 8u + (t & 7u)); }
__device__ __forceinline__ int patch_row(unsigned t) { return (int)((t >> 7) * 4u + ((t >> 3) & 3u)); }

// A thread produces RPT consecutive rows of one destination column: the per-pixel index / pointer set-up and the column terms
// cos*dx, sin*dx are paid once per RPT pixels (each product is still the reference's own rounded f32 product, so every source
// coordinate is bit-identical to the per-pixel formula).  Warp patch: 8 columns x (4 x RPT) rows; CTA tile: 32 x (8 x RPT).
constexpr int ROT_RPT = 8;   // measured on config 4: 8 rows per thread 1.66 ms / 128 frames, 4 rows 1.74 ms, 1 row 2.33 ms

// The general sampler, out of line: the Rgba8 bilinear fast path of rotate_kernel calls it only for samples that touch the image
// edge, and keeping eight inlined copies of it out of the unrolled row loop keeps that loop inside the instruction cache.
template <typename CT, int N, int METHOD, int BORDER_T>
__device__ __noinline__ void sample_general(const SrcView& img, float src_x, float src_y, const RotParams& p, const float* __restrict__ lut,
                                            Pix<CT, N>& val) {
    if (!interpolate<CT, N, METHOD, BORDER_T>(img, src_x, src_y, p.mb, p.mc, p.border, lut, val)) val = zero_px<CT, N>();
}

template <typename CT, int N, int METHOD, int BORDER_T>
__global__ void __launch_bounds__(256) rotate_kernel(SrcView img, unsigned long long src_image_pitch, CT* __restrict__ dst, size_t dst_stride,
                                                     unsigned long long dst_image_pitch, int dst_rows, int dst_cols, RotParams p,
                                                     const float* __restrict__ lut, unsigned slices) {
    const int c = blockIdx.x * 32 + patch_col(threadIdx.x);
    const int r0 = (ZB_LAYER_TILE(slices) * 8 + patch_row(threadIdx.x)) * ROT_RPT;
    if (c >= dst_cols || r0 >= dst_rows) return;
    const size_t frame = ZB_LAYER(slices);
    img.data = (const CT*)img.data + frame * src_image_pitch * N;
    CT* out = dst + (frame * dst_image_pitch + (size_t)r0 * dst_stride + (size_t)c) * N;
    const float x = (float)c;                                   // transforms.zig:199-209
    const float dx = x - p.rcx;
    const float cos_dx = p.cos_a * dx, sin_dx = p.sin_a * dx;   // the two products of this column
    if constexpr (BORDER_T == ZB_BORDER_ZERO && (METHOD == ZB_INTERP_BILINEAR || METHOD == ZB_INTERP_NEAREST)) {
        // Most of a rotated frame's bounding box is margin.  Every step of the coordinate formula is a monotone f32 operation of the
        // row, so the source coordinates of the rows in between lie between those of the first and the last row of this strip: if
        // both ends are outside the image on the same side (by more than the one-pixel reach of the sampler), the whole strip is zero.
        const int jl = min(ROT_RPT - 1, dst_rows - 1 - r0);
        const float dy0 = (float)r0 - p.rcy, dy1 = (float)(r0 + jl) - p.rcy;
        const float x0 = (cos_dx - p.sin_a * dy0) + p.cx, x1 = (cos_dx - p.sin_a * dy1) + p.cx;
        const float y0 = (sin_dx + p.cos_a * dy0) + p.cy, y1 = (sin_dx + p.cos_a * dy1) + p.cy;
        const float fc = (float)img.cols, fr = (float)img.rows;
        if (fmaxf(x0, x1) < -1.0f || fminf(x0, x1) >= fc || fmaxf(y0, y1) < -1.0f || fminf(y0, y1) >= fr) {
            const Pix<CT, N> z = zero_px<CT, N>();
            for (int j = 0; j <= jl; ++j) {
                store_px<CT, N>(out, 0, z);
                out += dst_stride * N;
            }
            return;
        }
    }
    // Rgba(u8), bilinear, frames below 2^21 pixels a side (config 4): an interior sample costs ONE float->int conversion per axis.
    // i = floor(512 * s) is exact (512 s is an exact product) and holds both floor(s) = i >> 9 and the reference's weight
    // @round(256 * frac) = ((i & 511) + 1) >> 1 (interpolation.zig:349-352; see frac_q8); offsets are 32-bit.  Samples that touch
    // the image edge take the general sampler below.
    constexpr bool kFastRgba8 = sizeof(CT) == 1 && N == 4 && METHOD == ZB_INTERP_BILINEAR;
    const bool fast_ok = kFastRgba8 && img.rows < (1 << 21) && img.cols < (1 << 21) && (unsigned long long)img.rows * img.stride < (1ull << 29);
    const float yf0 = (float)r0;
#pragma unroll
    for (int j = 0; j < ROT_RPT; ++j) {
        if (r0 + j >= dst_rows) break;
        const float y = kFastRgba8 ? yf0 + (float)j : (float)(r0 + j);   // exact either way
        const float dy = y - p.rcy;
        const float rotated_dx = cos_dx - p.sin_a * dy;
        const float rotated_dy = sin_dx + p.cos_a * dy;
        const float src_x = rotated_dx + p.cx;
        const float src_y = rotated_dy + p.cy;
        Pix<CT, N> val;
        bool done = false;
        if constexpr (kFastRgba8) {
            if (fast_ok && fabsf(src_x) < 2097152.0f && fabsf(src_y) < 2097152.0f) {
                const int ix = __float2int_rd(src_x * 512.0f), iy = __float2int_rd(src_y * 512.0f);
                const int left = ix >> 9, top = iy >> 9;
                if (BORDER_T == ZB_BORDER_ZERO && (left < -1 || left >= img.cols || top < -1 || top >= img.rows)) {
                    val.u = 0u;   // all four neighbours outside: .zero makes the sample 0 (the margin lanes of a partly covered strip)
                    done = true;
                } else if ((unsigned)left < (unsigned)(img.cols - 1) && (unsigned)top < (unsigned)(img.rows - 1)) {   // all four neighbours inside
                    const unsigned fx = (unsigned)((ix & 511) + 1) >> 1, fy = (unsigned)((iy & 511) + 1) >> 1;
                    const uint32_t* q = reinterpret_cast<const uint32_t*>(img.data) + (unsigned)top * (unsigned)img.stride + (unsigned)left;
                    const uint32_t* q2 = q + (unsigned)img.stride;
                    val.u = bilerp_rgba8(__ldg(q), __ldg(q + 1), __ldg(q2), __ldg(q2 + 1), fx, fy);
                    done = true;
                }
            }
        }
        if constexpr (kFastRgba8) {
            if (!done) sample_general<CT, N, METHOD, BORDER_T>(img, src_x, src_y, p, lut, val);
        } else {
            if (!interpolate<CT, N, METHOD, BORDER_T>(img, src_x, src_y, p.mb, p.mc, p.border, lut, val)) val = zero_px<CT, N>();
        }
        store_px<CT, N>(out, 0, val);
        out += dst_stride * N;
    }
}

// transforms.zig:385-462 as a gather over destination pixels
template <typename CT, int N>
__global__ void __launch_bounds__(256) rotate_orth_kernel(const CT* __restrict__ src, size_t src_stride, unsigned long long src_image_pitch,
                                                          int rows, int cols, CT* __restrict__ dst, size_t dst_stride,
                                                          unsigned long long dst_image_pitch, int dst_rows, int dst_cols, int kind,
                                                          unsigned slices) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int r = ZB_LAYER_TILE(slices) * 8 + (threadIdx.x >> 5);
    if (c >= dst_cols || r >= dst_rows) return;
    const size_t frame = ZB_LAYER(slices);
    src += frame * src_image_pitch * N;
    dst += frame * dst_image_pitch * N;
    const bool swap = (kind == 2 || kind == 4);
    const int content_rows = swap ? cols : rows, content_cols = swap ? rows : cols;
    const int offset_r = (dst_rows > content_rows ? dst_rows - content_rows : 0) / 2;
    const int offset_c = (dst_cols > content_cols ? dst_cols - content_cols : 0) / 2;
    const int rr = r - offset_r, cc = c - offset_c;
    if (rr >= 0 && rr < content_rows && cc >= 0 && cc < content_cols) {
        int sr, sc;
        switch (kind) {
            case 1: sr = rr; sc = cc; break;
            case 2: sc = cols - 1 - rr; sr = cc; break;              // new_r = cols-1-c, new_c = r
            case 3: sr = rows - 1 - rr; sc = cols - 1 - cc; break;
            default: sc = rr; sr = rows - 1 - cc; break;             // new_r = c, new_c = rows-1-r
        }
        store_px<CT, N>(dst, (size_t)r * dst_stride + c, load_px<CT, N>(src, (size_t)sr * src_stride + sc));
    } else if (offset_r != 0 || offset_c != 0) {
        store_px<CT, N>(dst, (size_t)r * dst_stride + c, zero_px<CT, N>());  // setBorder(inner, zeroes) only when an offset exists
    }
}

struct WarpParams {
    float m[9];
    int projective, method;
    float mb, mc;
};

template <typename CT, int N, int METHOD>
__global__ void __launch_bounds__(256) warp_kernel(SrcView img, CT* __restrict__ dst, size_t dst_stride, int dst_rows, int dst_cols,
                                                   WarpParams p, const float* __restrict__ lut) {
    const int c = blockIdx.x * 32 + patch_col(threadIdx.x);
    const int r = ZB_GRID_ROW() * 8 + patch_row(threadIdx.x);
    if (c >= dst_cols || r >= dst_rows) return;
    const float x = (float)c, y = (float)r;
    float sx, sy;
    if (p.projective) {  // geometry/transforms.zig:224-231 through SMatrix.gemm's scalar tail (SMatrix.zig:554-560)
        float d[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            float a = 0;
            a += p.m[3 * i + 0] * x;
            a += p.m[3 * i + 1] * y;
            a += p.m[3 * i + 2] * 1.0f;
            d[i] = 0.0f + 1.0f * a;
        }
        if (d[2] != 0) {
            const float s = 1 / d[2];
            d[0] = d[0] * s;
            d[1] = d[1] * s;
        }
        sx = d[0];
        sy = d[1];
    } else {  // :39-42 / :147-150
        float a0 = 0; a0 += p.m[0] * x; a0 += p.m[1] * y; a0 = 0.0f + 1.0f * a0;
        float a1 = 0; a1 += p.m[2] * x; a1 += p.m[3] * y; a1 = 0.0f + 1.0f * a1;
        sx = a0 + p.m[4];
        sy = a1 + p.m[5];
    }
    Pix<CT, N> val;
    if (!interpolate<CT, N, METHOD, ZB_BORDER_MIRROR>(img, sx, sy, p.mb, p.mc, ZB_BORDER_MIRROR, lut, val)) val = zero_px<CT, N>();
    store_px<CT, N>(dst, (size_t)r * dst_stride + c, val);
}

template <typename CT, int N>
int rotate_typed(const zb_image* src, unsigned long long spitch, zb_image* dst, unsigned long long dpitch, uint32_t n, float angle,
                 float cos_a, float sin_a, int method, float mb, float mc, int border, const float* lut, cudaStream_t s) {
    const int cls = rotate_class(angle);
    dim3 grid;
    unsigned slices;
    int rc;
    if (cls != 0) {
        if ((rc = layered_row_grid(div_up(dst->cols, 32), div_up(dst->rows, 8), n, &grid, &slices))) return rc;
        t_last_kernel = "rotate_orthogonal";
        rotate_orth_kernel<CT, N><<<grid, 256, 0, s>>>((const CT*)src->data, (size_t)src->stride, spitch, (int)src->rows, (int)src->cols,
                                                       (CT*)dst->data, (size_t)dst->stride, dpitch, (int)dst->rows, (int)dst->cols, cls,
                                                       slices);
        ZB_LAUNCHED();
        return ZB_OK;
    }
    RotParams p;
    p.cos_a = cos_a;
    p.sin_a = sin_a;
    p.cx = (float)src->cols / 2.0f;   // image.zig:322-327
    p.cy = (float)src->rows / 2.0f;
    const float offset_x = ((float)dst->cols - (float)src->cols) / 2.0f;   // transforms.zig:193-197
    const float offset_y = ((float)dst->rows - (float)src->rows) / 2.0f;
    p.rcx = p.cx + offset_x;
    p.rcy = p.cy + offset_y;
    p.method = method; p.border = border; p.mb = mb; p.mc = mc;
    if constexpr (sizeof(CT) == 1 && N == 4) {   // Rgba(u8), bilinear, .zero (config 4): shared-memory source tiles, zb_rotate_tile.cu
        if (g_tune_rotate_tile.load()) {
            rc = rotate_tile_rgba8(src, spitch, dst, dpitch, n, p, s);
            if (rc != ZB_ERR_UNSUPPORTED) return rc;
        }
    }
    if ((rc = layered_row_grid(div_up(dst->cols, 32), div_up(dst->rows, 8 * ROT_RPT), n, &grid, &slices))) return rc;
    SrcView v{src->data, (int)src->rows, (int)src->cols, src->stride};
    t_last_kernel = "rotate_gather";
    return dispatch_method(method, [&](auto m) -> int {
        constexpr int M = decltype(m)::value;
        // the default front-end combination (bilinear / nearest with .zero, python binding transforms.zig:250-251) gets a
        // kernel with the border folded at compile time; everything else keeps it a runtime value
        constexpr int BT = (M == ZB_INTERP_BILINEAR || M == ZB_INTERP_NEAREST) ? ZB_BORDER_ZERO : -1;
        CT* dp = (CT*)dst->data;
        const size_t ds = (size_t)dst->stride;
        const int dr = (int)dst->rows, dc = (int)dst->cols;
        if ((M == ZB_INTERP_BILINEAR || M == ZB_INTERP_NEAREST) && border == ZB_BORDER_ZERO)
            rotate_kernel<CT, N, M, BT><<<grid, 256, 0, s>>>(v, spitch, dp, ds, dpitch, dr, dc, p, lut, slices);
        else
            rotate_kernel<CT, N, M, -1><<<grid, 256, 0, s>>>(v, spitch, dp, ds, dpitch, dr, dc, p, lut, slices);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}

int rotate_dispatch(const zb_image* src, unsigned long long spitch, zb_image* dst, unsigned long long dpitch, uint32_t n, int pixfmt,
                    float angle, float cos_a, float sin_a, int method, float mb, float mc, int border, cudaStream_t s) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (method < ZB_INTERP_NEAREST || method > ZB_INTERP_LANCZOS) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    if (dst->rows == 0 || dst->cols == 0 || n == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const float* lut = nullptr;
    if (method == ZB_INTERP_LANCZOS && (rc = lanczos_lut_device(&lut, s))) return rc;
    switch (pixfmt) {
        case ZB_PIX_U8: return rotate_typed<uint8_t, 1>(src, spitch, dst, dpitch, n, angle, cos_a, sin_a, method, mb, mc, border, lut, s);
        case ZB_PIX_F32: return rotate_typed<float, 1>(src, spitch, dst, dpitch, n, angle, cos_a, sin_a, method, mb, mc, border, lut, s);
        case ZB_PIX_RGB8: return rotate_typed<uint8_t, 3>(src, spitch, dst, dpitch, n, angle, cos_a, sin_a, method, mb, mc, border, lut, s);
        case ZB_PIX_RGBA8: return rotate_typed<uint8_t, 4>(src, spitch, dst, dpitch, n, angle, cos_a, sin_a, method, mb, mc, border, lut, s);
        case ZB_PIX_RGBAF32: return rotate_typed<float, 4>(src, spitch, dst, dpitch, n, angle, cos_a, sin_a, method, mb, mc, border, lut, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

template <typename CT, int N>
int warp_typed(const zb_image* src, zb_image* dst, const WarpParams& p, const float* lut, cudaStream_t s) {
    SrcView v{src->data, (int)src->rows, (int)src->cols, src->stride};
    const dim3 grid = row_grid(div_up(dst->cols, 32), div_up(dst->rows, 8));
    return dispatch_method(p.method, [&](auto m) -> int {
        warp_kernel<CT, N, decltype(m)::value><<<grid, 256, 0, s>>>(v, (CT*)dst->data, (size_t)dst->stride, (int)dst->rows, (int)dst->cols, p, lut);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}

int warp_dispatch(const zb_image* src, zb_image* dst, int pixfmt, int kind, const float* m, int method, float mb, float mc, cudaStream_t s) {
    if (!src || !dst || !m) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (kind < ZB_XFORM_SIMILARITY || kind > ZB_XFORM_PROJECTIVE) return ZB_ERR_INVALID_ARGUMENT;
    if (method < ZB_INTERP_NEAREST || method > ZB_INTERP_LANCZOS) return ZB_ERR_INVALID_ARGUMENT;
    if (dst->rows == 0 || dst->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    WarpParams p;
    memset(&p, 0, sizeof(p));
    p.projective = kind == ZB_XFORM_PROJECTIVE;
    memcpy(p.m, m, (p.projective ? 9 : 6) * sizeof(float));
    p.method = method; p.mb = mb; p.mc = mc;
    const float* lut = nullptr;
    if (method == ZB_INTERP_LANCZOS && (rc = lanczos_lut_device(&lut, s))) return rc;
    t_last_kernel = "warp_gather";
    switch (pixfmt) {
        case ZB_PIX_U8: return warp_typed<uint8_t, 1>(src, dst, p, lut, s);
        case ZB_PIX_F32: return warp_typed<float, 1>(src, dst, p, lut, s);
        case ZB_PIX_RGB8: return warp_typed<uint8_t, 3>(src, dst, p, lut, s);
        case ZB_PIX_RGBA8: return warp_typed<uint8_t, 4>(src, dst, p, lut, s);
        case ZB_PIX_RGBAF32: return warp_typed<float, 4>(src, dst, p, lut, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

// ---- Image.extract (transforms.zig:232-283) and its copyRect fast path (:465-518) ---------------------------------------------
struct ExtractParams {
    float rl, rt, width, height, cx, cy, cos_a, sin_a, frows1, fcols1;   // frows1 = rows - 1 as f32
    int copy_rect, rect_top, rect_left;                                   // fast path: integer shift + border
    int border, method;
    float mb, mc;
};

template <typename CT, int N, int METHOD>
__global__ void __launch_bounds__(256) extract_kernel(SrcView img, CT* __restrict__ dst, size_t dst_stride, int dst_rows, int dst_cols,
                                                      ExtractParams p, const float* __restrict__ lut) {
    const int c = blockIdx.x * 32 + patch_col(threadIdx.x);
    const int r = ZB_GRID_ROW() * 8 + patch_row(threadIdx.x);
    if (c >= dst_cols || r >= dst_rows) return;
    Pix<CT, N> val;
    if (p.copy_rect) {   // out(r, c) = self(resolve(r + top), resolve(c + left)) or zero
        const int sr = resolve_index(r + p.rect_top, img.rows, p.border);
        const int sc = resolve_index(c + p.rect_left, img.cols, p.border);
        val = (sr < 0 || sc < 0) ? zero_px<CT, N>() : load_px<CT, N>((const CT*)img.data, (size_t)sr * img.stride + (size_t)sc);
    } else {             // normalised mapping, rotation by +angle around the rect centre (unfused f32, the reference's order)
        const float ty = dst_rows == 1 ? 0.5f : (float)r / p.frows1;
        const float y_rect = p.rt + ty * p.height;
        const float tx = dst_cols == 1 ? 0.5f : (float)c / p.fcols1;
        const float x_rect = p.rl + tx * p.width;
        const float dx = x_rect - p.cx, dy = y_rect - p.cy;
        const float src_x = p.cx + p.cos_a * dx - p.sin_a * dy;
        const float src_y = p.cy + p.sin_a * dx + p.cos_a * dy;
        if (!interpolate<CT, N, METHOD, -1>(img, src_x, src_y, p.mb, p.mc, p.border, lut, val)) val = zero_px<CT, N>();
    }
    store_px<CT, N>(dst, (size_t)r * dst_stride + c, val);
}

template <typename CT, int N>
int extract_typed(const zb_image* src, zb_image* dst, const ExtractParams& p, const float* lut, cudaStream_t s) {
    SrcView v{src->data, (int)src->rows, (int)src->cols, src->stride};
    const dim3 grid = row_grid(div_up(dst->cols, 32), div_up(dst->rows, 8));
    return dispatch_method(p.method, [&](auto m) -> int {
        extract_kernel<CT, N, decltype(m)::value><<<grid, 256, 0, s>>>(v, (CT*)dst->data, (size_t)dst->stride, (int)dst->rows, (int)dst->cols, p, lut);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}

int extract_dispatch(const zb_image* src, zb_image* dst, int pixfmt, float rl, float rt, float rr, float rb, float angle, float cos_a,
                     float sin_a, int method, float mb, float mc, int border, cudaStream_t s) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (method < ZB_INTERP_NEAREST || method > ZB_INTERP_LANCZOS) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    if (dst->rows == 0 || dst->cols == 0) return ZB_OK;   // :233
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (src->rows == 0 || src->cols == 0) {   // every sample resolves to null -> zeroes (tests/transforms.zig:411-424)
        ZB_CUDA(cudaMemset2DAsync(dst->data, dst->stride * pixel_bytes(pixfmt), 0, (size_t)dst->cols * pixel_bytes(pixfmt), dst->rows, s));
        return ZB_OK;
    }
    ExtractParams p;
    memset(&p, 0, sizeof(p));
    const float frows = (float)dst->rows, fcols = (float)dst->cols;
    p.rl = rl; p.rt = rt;
    p.width = rl >= rr ? 0.0f : rr - rl;   // Rectangle(f32).width / height return 0 for an inverted rect (Rectangle.zig:76-93)
    p.height = rt >= rb ? 0.0f : rb - rt;
    const float epsilon = 1e-6f;
    if (std::fabs(angle) < epsilon && std::fabs(p.width - fcols) < epsilon && std::fabs(p.height - frows) < epsilon) {   // :241-250
        p.copy_rect = 1;
        p.rect_top = (int)std::round(rt);
        p.rect_left = (int)std::round(rl);
    }
    p.cx = (rl + rr) * 0.5f; p.cy = (rt + rb) * 0.5f;
    p.cos_a = cos_a; p.sin_a = sin_a;
    p.frows1 = frows - 1; p.fcols1 = fcols - 1;
    p.border = border; p.method = method; p.mb = mb; p.mc = mc;
    const float* lut = nullptr;
    if (method == ZB_INTERP_LANCZOS && (rc = lanczos_lut_device(&lut, s))) return rc;
    t_last_kernel = p.copy_rect ? "extract_copy_rect" : "extract_gather";
    switch (pixfmt) {
        case ZB_PIX_U8: return extract_typed<uint8_t, 1>(src, dst, p, lut, s);
        case ZB_PIX_F32: return extract_typed<float, 1>(src, dst, p, lut, s);
        case ZB_PIX_RGB8: return extract_typed<uint8_t, 3>(src, dst, p, lut, s);
        case ZB_PIX_RGBA8: return extract_typed<uint8_t, 4>(src, dst, p, lut, s);
        case ZB_PIX_RGBAF32: return extract_typed<float, 4>(src, dst, p, lut, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

// ---- Image.insert (transforms.zig:293-376), same pixel type: the complement of extract; Rgba(u8) samples composite under a blend
// mode (image.zig:67-95 assignPixel), every other pixel type assigns -----------------------------------------------------------

template <typename CT, int N, int METHOD>
__global__ void __launch_bounds__(256) insert_kernel(SrcView source, CT* __restrict__ self, size_t self_stride, InsertParams p,
                                                     const float* __restrict__ lut) {
    const int wc = blockIdx.x * 32 + patch_col(threadIdx.x);
    const int wr = ZB_GRID_ROW() * 8 + patch_row(threadIdx.x);
    if (wc >= p.n_c || wr >= p.n_r) return;
    const int r = p.min_r + wr, c = p.min_c + wc;   // destination pixel
    Pix<CT, N> val;
    if (p.copy_rect) {
        val = load_px<CT, N>((const CT*)source.data, (size_t)(r - p.dst_top) * source.stride + (size_t)(c - p.dst_left));
    } else {
        const float dy = (float)r - p.cy, dx = (float)c - p.cx;
        const float rect_x = p.cos_a * dx + p.sin_a * dy;        // inverse rotation into rectangle space
        const float rect_y = -p.sin_a * dx + p.cos_a * dy;
        if (fabsf(rect_x) > p.half_w || fabsf(rect_y) > p.half_h) return;
        const float norm_x = (rect_x + p.half_w) * p.inv_w;
        const float norm_y = (rect_y + p.half_h) * p.inv_h;
        const float src_x = p.src_cols == 1 ? 0.0f : norm_x * p.fcols1;
        const float src_y = p.src_rows == 1 ? 0.0f : norm_y * p.frows1;
        if (!interpolate<CT, N, METHOD, ZB_BORDER_MIRROR>(source, src_x, src_y, p.mb, p.mc, ZB_BORDER_MIRROR, lut, val)) return;
    }
    if constexpr (sizeof(CT) == 1 && N == 4) {
        if (p.blend != ZB_BLEND_NONE) val.u = blend_rgba8(load_px<CT, N>(self, (size_t)r * self_stride + c).u, val.u, p.blend);
    }
    store_px<CT, N>(self, (size_t)r * self_stride + c, val);
}

template <typename CT, int N>
int insert_typed(zb_image* self, const zb_image* source, const InsertParams& p, const float* lut, cudaStream_t s) {
    SrcView v{source->data, (int)source->rows, (int)source->cols, source->stride};
    const dim3 grid = row_grid(div_up(p.n_c, 32), div_up(p.n_r, 8));
    return dispatch_method(p.method, [&](auto m) -> int {
        insert_kernel<CT, N, decltype(m)::value><<<grid, 256, 0, s>>>(v, (CT*)self->data, (size_t)self->stride, p, lut);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}

int insert_dispatch(zb_image* self, const zb_image* source, int pixfmt, float rl, float rt, float rr, float rb, float angle, float cos_a,
                    float sin_a, int method, float mb, float mc, int blend, cudaStream_t s) {
    if (!self || !source) return ZB_ERR_INVALID_ARGUMENT;
    if (blend < ZB_BLEND_NONE || blend > ZB_BLEND_EXCLUSION) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (method < ZB_INTERP_NEAREST || method > ZB_INTERP_LANCZOS) return ZB_ERR_INVALID_ARGUMENT;
    if (source->rows == 0 || source->cols == 0) return ZB_OK;   // :294
    if (self->rows == 0 || self->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    InsertParams p;
    if (!insert_plan(self, source, rl, rt, rr, rb, angle, cos_a, sin_a, method, mb, mc, blend, p)) return ZB_OK;   // nothing to write
    const float* lut = nullptr;
    if (method == ZB_INTERP_LANCZOS && (rc = lanczos_lut_device(&lut, s))) return rc;
    t_last_kernel = p.copy_rect ? "insert_copy_rect" : "insert_gather";
    switch (pixfmt) {
        case ZB_PIX_U8: return insert_typed<uint8_t, 1>(self, source, p, lut, s);
        case ZB_PIX_F32: return insert_typed<float, 1>(self, source, p, lut, s);
        case ZB_PIX_RGB8: return insert_typed<uint8_t, 3>(self, source, p, lut, s);
        case ZB_PIX_RGBA8: return insert_typed<uint8_t, 4>(self, source, p, lut, s);
        case ZB_PIX_RGBAF32: return insert_typed<float, 4>(self, source, p, lut, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

}  // namespace

// interpolation.zig:256-267: lut[i] = lanczosKernel(i / (1024/3), 3) in f32, computed on the host
int lanczos_lut_device(const float** out, cudaStream_t s) {
    static std::mutex mu;
    static float* dev_lut[64] = {nullptr};    // published once the upload has completed: any stream may read it afterwards
    static float* dev_alloc[64] = {nullptr};
    int dev = 0;
    ZB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);
    if (!dev_lut[dev]) {
        float h[1025];
        const float step = 1024.0f / 3.0f;
        for (int i = 0; i < 1025; ++i) {
            const float x = (float)i / step;
            float v;
            if (x == 0) v = 1;
            else if (std::fabs(x) >= 3.0f) v = 0;
            else {
                const float pi_x = 3.14159265358979323846f * x;
                const float pi_x_over_a = pi_x / 3.0f;
                v = (3.0f * std::sin(pi_x) * std::sin(pi_x_over_a)) / (pi_x * pi_x);
            }
            h[i] = v;
        }
        // on the caller's stream, synchronised before publishing (a plain cudaMemcpy from pageable memory would wait for the
        // legacy NULL stream and may return before the copy lands)
        if (!dev_alloc[dev]) ZB_CUDA(cudaMalloc(&dev_alloc[dev], sizeof(h)));
        ZB_CUDA(cudaMemcpyAsync(dev_alloc[dev], h, sizeof(h), cudaMemcpyHostToDevice, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        dev_lut[dev] = dev_alloc[dev];
    }
    *out = dev_lut[dev];
    return ZB_OK;
}

}  // namespace zb

using namespace zb;

extern "C" {

int zb_rotate_bounds(uint32_t rows, uint32_t cols, float angle, uint32_t* out_rows, uint32_t* out_cols) {
    if (!out_rows || !out_cols) return ZB_ERR_INVALID_ARGUMENT;
    const int cls = rotate_class(angle);
    if (cls == 1 || cls == 3) { *out_rows = rows; *out_cols = cols; return ZB_OK; }
    if (cls == 2 || cls == 4) { *out_rows = cols; *out_cols = rows; return ZB_OK; }
    const float cos_abs = std::fabs(std::cos(angle)), sin_abs = std::fabs(std::sin(angle));  // transforms.zig:139-148
    const float w = (float)cols, h = (float)rows;
    const float new_w = w * cos_abs + h * sin_abs;
    const float new_h = h * cos_abs + w * sin_abs;
    *out_cols = (uint32_t)std::ceil(new_w);
    *out_rows = (uint32_t)std::ceil(new_h);
    return ZB_OK;
}

int zb_rotate_into_cs(const zb_image* src, zb_image* dst, int pixfmt, float angle, float cos_a, float sin_a, int method, float mb,
                      float mc, int border, zb_stream s) {
    return rotate_dispatch(src, 0, dst, 0, 1, pixfmt, angle, cos_a, sin_a, method, mb, mc, border, (cudaStream_t)s);
}

int zb_rotate_into(const zb_image* src, zb_image* dst, int pixfmt, float angle, int method, float mb, float mc, int border, zb_stream s) {
    return rotate_dispatch(src, 0, dst, 0, 1, pixfmt, angle, std::cos(angle), std::sin(angle), method, mb, mc, border, (cudaStream_t)s);
}

int zb_rotate_into_batch(const zb_image* src0, uint64_t src_image_pitch_px, zb_image* dst0, uint64_t dst_image_pitch_px, uint32_t n_images,
                         int pixfmt, float angle, float cos_a, float sin_a, int method, float mb, float mc, int border, zb_stream s) {
    if (n_images > 65535) return ZB_ERR_INVALID_ARGUMENT;
    return rotate_dispatch(src0, src_image_pitch_px, dst0, dst_image_pitch_px, n_images, pixfmt, angle, cos_a, sin_a, method, mb, mc, border,
                           (cudaStream_t)s);
}

int zb_insert(zb_image* self, const zb_image* source, int pixfmt, float rect_l, float rect_t, float rect_r, float rect_b, float angle,
              float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, zb_stream s) {
    return insert_dispatch(self, source, pixfmt, rect_l, rect_t, rect_r, rect_b, angle, cos_a, sin_a, method, mitchell_b, mitchell_c,
                           ZB_BLEND_NONE, (cudaStream_t)s);
}

int zb_insert_blend(zb_image* self, const zb_image* source, int pixfmt, float rect_l, float rect_t, float rect_r, float rect_b, float angle,
                    float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, int blend_mode, zb_stream s) {
    return insert_dispatch(self, source, pixfmt, rect_l, rect_t, rect_r, rect_b, angle, cos_a, sin_a, method, mitchell_b, mitchell_c,
                           blend_mode, (cudaStream_t)s);
}

int zb_extract(const zb_image* src, zb_image* dst, int pixfmt, float rect_l, float rect_t, float rect_r, float rect_b, float angle,
               float cos_a, float sin_a, int method, float mitchell_b, float mitchell_c, int border, zb_stream s) {
    return extract_dispatch(src, dst, pixfmt, rect_l, rect_t, rect_r, rect_b, angle, cos_a, sin_a, method, mitchell_b, mitchell_c, border,
                            (cudaStream_t)s);
}

int zb_warp(const zb_image* src, zb_image* dst, int pixfmt, int xform_kind, const float* m, int method, float mb, float mc, zb_stream s) {
    return warp_dispatch(src, dst, pixfmt, xform_kind, m, method, mb, mc, (cudaStream_t)s);
}

int zb_host_rotate_into(const zb_image* src, zb_image* dst, int pixfmt, float angle, int method, float mb, float mc, int border) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    HostStage st;
    int rc;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = zb_rotate_into(&st.dsrc, &st.ddst, pixfmt, angle, method, mb, mc, border, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

int zb_host_warp(const zb_image* src, zb_image* dst, int pixfmt, int xform_kind, const float* m, int method, float mb, float mc) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    HostStage st;
    int rc;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = zb_warp(&st.dsrc, &st.ddst, pixfmt, xform_kind, m, method, mb, mc, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

}  // extern "C"
