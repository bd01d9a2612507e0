// zb_conv_generic.cu -- general separable / dense convolution kernels: every pixel format, border
// mode, tap count and stride.  Two-pass (temp plane in HBM) for the separable case, i.e. the same
// data flow as the reference (convolution.zig:441-647); arithmetic is bit-exact with it:
//   f32: acc = acc + px*k with separately rounded mul and add, taps ascending, |k| < 1e-10 taps
//        skipped only for interior outputs (convolution.zig:459-467,541 vs :526-530);
//   u8:  Q8 taps round(k*256) (:303-309), i32 temp saturated (:495-513), divClampU8(65536) (:485);
//        accumulators are i32 when the host proves they cannot overflow, i64 otherwise.
// Interleaved Rgb/Rgba u8 pixels are filtered in place per channel (tap offset = CH elements); the
// reference's split -> plane -> merge (:358,:430) computes the same per-channel values.
// The fused single-pass kernel for the headline format lives in zb_conv_fused.cu.
#include "zb_conv.h"
#include "zb_device.cuh"

namespace zb {

constexpr int kThreads = 256;

template <typename T> struct IsFloat { static constexpr bool value = false; };
template <> struct IsFloat<float> { static constexpr bool value = true; };

// ---------------------------------------------------------------------------------------------
// Horizontal pass: src (strided, CH interleaved channels) -> tmp (contiguous rows x cols*CH)
// ---------------------------------------------------------------------------------------------
template <typename SrcT, typename TmpT, typename AccT, typename KT, int CH>
__global__ void __launch_bounds__(kThreads) sep_h_kernel(const SrcT* __restrict__ src, size_t src_row_el, TmpT* __restrict__ tmp,
                                                         int rows, int cols, const KT* __restrict__ taps_g, int nx, int border) {
    extern __shared__ unsigned char smem_raw[];
    KT* taps = reinterpret_cast<KT*>(smem_raw);
    for (int i = threadIdx.x; i < nx; i += blockDim.x) taps[i] = taps_g[i];
    __syncthreads();
    const int r = ZB_GRID_ROW();
    const int e = blockIdx.x * blockDim.x + threadIdx.x;  // element within the row
    const int w = cols * CH;
    if (e >= w || r >= rows) return;
    const int c = e / CH, k = e - c * CH;
    const int half = nx / 2;
    const SrcT* row = src + (size_t)r * src_row_el;
    const bool interior = (cols > 2 * half) && c >= half && c < cols - half;
    AccT acc = 0;
    if (interior) {
        const SrcT* p = row + (size_t)(c - half) * CH + k;
        for (int i = 0; i < nx; ++i) {
            const KT kv = taps[i];
            if constexpr (IsFloat<KT>::value) {
                if (fabsf(kv) < 1e-10f) continue;
                acc = mul_add_unfused((float)p[(size_t)i * CH], kv, acc);
            } else {
                acc += (AccT)p[(size_t)i * CH] * (AccT)kv;
            }
        }
    } else {
        for (int i = 0; i < nx; ++i) {
            const int ci = resolve_index(c + i - half, cols, border);
            if constexpr (IsFloat<KT>::value) {
                const float pv = ci < 0 ? 0.0f : (float)row[(size_t)ci * CH + k];
                acc = mul_add_unfused(pv, taps[i], acc);
            } else {
                const AccT pv = ci < 0 ? (AccT)0 : (AccT)row[(size_t)ci * CH + k];
                acc += pv * (AccT)taps[i];
            }
        }
    }
    if constexpr (IsFloat<KT>::value) {
        tmp[(size_t)r * w + e] = acc;
    } else if constexpr (sizeof(AccT) == 8) {
        const AccT lo = -2147483648LL, hi = 2147483647LL;
        tmp[(size_t)r * w + e] = (TmpT)(acc < lo ? lo : (acc > hi ? hi : acc));
    } else {
        tmp[(size_t)r * w + e] = (TmpT)acc;
    }
}

// ---------------------------------------------------------------------------------------------
// Vertical pass: tmp (contiguous) -> dst (strided)
// ---------------------------------------------------------------------------------------------
template <typename DstT, typename TmpT, typename AccT, typename KT, int CH>
__global__ void __launch_bounds__(kThreads) sep_v_kernel(const TmpT* __restrict__ tmp, DstT* __restrict__ dst, size_t dst_row_el,
                                                         int rows, int cols, const KT* __restrict__ taps_g, int ny, int border) {
    extern __shared__ unsigned char smem_raw[];
    KT* taps = reinterpret_cast<KT*>(smem_raw);
    for (int i = threadIdx.x; i < ny; i += blockDim.x) taps[i] = taps_g[i];
    __syncthreads();
    const int r = ZB_GRID_ROW();
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int w = cols * CH;
    if (e >= w || r >= rows) return;
    const int half = ny / 2;
    const bool interior = (rows > 2 * half) && r >= half && r < rows - half;
    AccT acc = 0;
    if (interior) {
        const TmpT* p = tmp + (size_t)(r - half) * w + e;
        for (int i = 0; i < ny; ++i) {
            const KT kv = taps[i];
            if constexpr (IsFloat<KT>::value) {
                if (fabsf(kv) < 1e-10f) continue;
                acc = mul_add_unfused(p[(size_t)i * w], kv, acc);
            } else {
                acc += (AccT)p[(size_t)i * w] * (AccT)kv;
            }
        }
    } else {
        for (int i = 0; i < ny; ++i) {
            const int ri = resolve_index(r + i - half, rows, border);
            if constexpr (IsFloat<KT>::value) {
                const float pv = ri < 0 ? 0.0f : tmp[(size_t)ri * w + e];
                acc = mul_add_unfused(pv, taps[i], acc);
            } else {
                const AccT pv = ri < 0 ? (AccT)0 : (AccT)tmp[(size_t)ri * w + e];
                acc += pv * (AccT)taps[i];
            }
        }
    }
    if constexpr (IsFloat<KT>::value) dst[(size_t)r * dst_row_el + e] = acc;
    else dst[(size_t)r * dst_row_el + e] = div_clamp_u8<AccT>(acc, (AccT)65536);
}

// ---------------------------------------------------------------------------------------------
// Dense kh x kw correlation (no kernel flip), convolution.zig:113-193.  One thread per PIXEL: the border
// resolution and the tap loop are shared by the CH channels, RGBA pixels move as one 32-bit word.
// ---------------------------------------------------------------------------------------------
template <typename PixT, int CH>
__device__ __forceinline__ void load_channels(const PixT* __restrict__ p, float* v) {
#pragma unroll
    for (int k = 0; k < CH; ++k) v[k] = (float)p[k];
}
template <typename PixT, int CH>
__device__ __forceinline__ void load_channels(const PixT* __restrict__ p, int* v) {
    if constexpr (CH == 4 && sizeof(PixT) == 1) {
        const uchar4 q = *reinterpret_cast<const uchar4*>(p);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
        for (int k = 0; k < CH; ++k) v[k] = (int)p[k];
    }
}
template <typename PixT, int CH>
__device__ __forceinline__ void load_channels(const PixT* __restrict__ p, long long* v) {
#pragma unroll
    for (int k = 0; k < CH; ++k) v[k] = (long long)p[k];
}

template <typename PixT, typename AccT, typename KT, int CH>
__global__ void __launch_bounds__(kThreads) conv2d_kernel(const PixT* __restrict__ src, size_t src_row_el, PixT* __restrict__ dst,
                                                          size_t dst_row_el, int rows, int cols, const KT* __restrict__ taps_g,
                                                          int kh, int kw, int border) {
    extern __shared__ unsigned char smem_raw[];
    KT* taps = reinterpret_cast<KT*>(smem_raw);
    for (int i = threadIdx.x; i < kh * kw; i += blockDim.x) taps[i] = taps_g[i];
    __syncthreads();
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int r = ZB_GRID_ROW() * 8 + (threadIdx.x >> 5);
    if (c >= cols || r >= rows) return;
    const int half_h = kh / 2, half_w = kw / 2;
    const bool interior = r >= half_h && r + half_h < rows && c >= half_w && c + half_w < cols;
    AccT acc[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) acc[k] = 0;
    for (int ky = 0; ky < kh; ++ky) {
        int ry = r + ky - half_h;
        if (!interior) ry = resolve_index(ry, rows, border);
        for (int kx = 0; kx < kw; ++kx) {
            int cx = c + kx - half_w;
            if (!interior) cx = resolve_index(cx, cols, border);
            const KT kv = taps[ky * kw + kx];
            AccT pv[CH];
            if (ry < 0 || cx < 0) {
#pragma unroll
                for (int k = 0; k < CH; ++k) pv[k] = 0;
            } else {
                load_channels<PixT, CH>(src + (size_t)ry * src_row_el + (size_t)cx * CH, pv);
            }
#pragma unroll
            for (int k = 0; k < CH; ++k) {
                if constexpr (IsFloat<KT>::value) acc[k] = mul_add_unfused(pv[k], kv, acc[k]);
                else acc[k] += pv[k] * (AccT)kv;
            }
        }
    }
    PixT* out = dst + (size_t)r * dst_row_el + (size_t)c * CH;
    if constexpr (IsFloat<KT>::value) {
#pragma unroll
        for (int k = 0; k < CH; ++k) out[k] = acc[k];
    } else if constexpr (CH == 4) {
        *reinterpret_cast<uchar4*>(out) = make_uchar4(div_clamp_u8<AccT>(acc[0], (AccT)256), div_clamp_u8<AccT>(acc[1], (AccT)256),
                                                      div_clamp_u8<AccT>(acc[2], (AccT)256), div_clamp_u8<AccT>(acc[3], (AccT)256));
    } else {
#pragma unroll
        for (int k = 0; k < CH; ++k) out[k] = div_clamp_u8<AccT>(acc[k], (AccT)256);
    }
}

// ---------------------------------------------------------------------------------------------
// Host-side launchers
// ---------------------------------------------------------------------------------------------
template <typename PixT, typename TmpT, typename AccH, typename AccV, typename KT, int CH>
static int launch_sep(const zb_image* src, zb_image* dst, const KT* d_kx, int nx, const KT* d_ky, int ny, int border, void* tmp,
                      cudaStream_t s) {
    const int rows = (int)src->rows, cols = (int)src->cols;
    const int w = cols * CH;
    const dim3 grid = row_grid(div_up(w, kThreads), (size_t)rows);
    sep_h_kernel<PixT, TmpT, AccH, KT, CH><<<grid, kThreads, nx * sizeof(KT), s>>>((const PixT*)src->data, (size_t)src->stride * CH,
                                                                                   (TmpT*)tmp, rows, cols, d_kx, nx, border);
    ZB_LAUNCHED();
    sep_v_kernel<PixT, TmpT, AccV, KT, CH><<<grid, kThreads, ny * sizeof(KT), s>>>((const TmpT*)tmp, (PixT*)dst->data,
                                                                                   (size_t)dst->stride * CH, rows, cols, d_ky, ny, border);
    ZB_LAUNCHED();
    return ZB_OK;
}

template <int CH>
static int sep_u8_dispatch(const zb_image* src, zb_image* dst, const int32_t* d_kx, int nx, const int32_t* d_ky, int ny, int border,
                           void* tmp, bool h32, bool v32, cudaStream_t s) {
    if (h32 && v32) return launch_sep<uint8_t, int32_t, int32_t, int32_t, int32_t, CH>(src, dst, d_kx, nx, d_ky, ny, border, tmp, s);
    if (h32) return launch_sep<uint8_t, int32_t, int32_t, long long, int32_t, CH>(src, dst, d_kx, nx, d_ky, ny, border, tmp, s);
    return launch_sep<uint8_t, int32_t, long long, long long, int32_t, CH>(src, dst, d_kx, nx, d_ky, ny, border, tmp, s);
}

int conv_separable_generic(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny,
                           int border, cudaStream_t s) {
    const int ch = channels_of(pixfmt);
    const size_t n_el = (size_t)src->rows * src->cols * ch;
    if (nx > kMaxTaps || ny > kMaxTaps) return ZB_ERR_UNSUPPORTED;
    Scratch taps, tmp;
    int rc;
    if ((rc = taps.alloc((size_t)(nx + ny) * 4, s))) return rc;
    if ((rc = tmp.alloc(n_el * 4, s))) return rc;
    if (is_float_fmt(pixfmt)) {
        ZB_CUDA(cudaMemcpyAsync(taps.p, kx, (size_t)nx * 4, cudaMemcpyHostToDevice, s));
        ZB_CUDA(cudaMemcpyAsync((float*)taps.p + nx, ky, (size_t)ny * 4, cudaMemcpyHostToDevice, s));
        const float* dkx = (const float*)taps.p;
        const float* dky = dkx + nx;
        t_last_kernel = "sep_generic_f32";
        if (ch == 1) return launch_sep<float, float, float, float, float, 1>(src, dst, dkx, nx, dky, ny, border, tmp.p, s);
        return launch_sep<float, float, float, float, float, 4>(src, dst, dkx, nx, dky, ny, border, tmp.p, s);
    }
    // u8 family: Q8 taps on the host (convolution.zig:303-309), overflow analysis for the accumulators
    int32_t ki[2 * kMaxTaps];
    int64_t sax = 0, say = 0;
    for (int i = 0; i < nx; ++i) { ki[i] = (int32_t)roundf(kx[i] * 256.0f); sax += llabs((long long)ki[i]); }
    for (int i = 0; i < ny; ++i) { ki[nx + i] = (int32_t)roundf(ky[i] * 256.0f); say += llabs((long long)ki[nx + i]); }
    const bool h32 = sax * 255 < 2147483647LL;
    const bool v32 = h32 && (sax * 255) * say < 2147483647LL;
    ZB_CUDA(cudaMemcpyAsync(taps.p, ki, (size_t)(nx + ny) * 4, cudaMemcpyHostToDevice, s));
    const int32_t* dkx = (const int32_t*)taps.p;
    const int32_t* dky = dkx + nx;
    t_last_kernel = "sep_generic_u8";
    switch (ch) {
        case 1: return sep_u8_dispatch<1>(src, dst, dkx, nx, dky, ny, border, tmp.p, h32, v32, s);
        case 3: return sep_u8_dispatch<3>(src, dst, dkx, nx, dky, ny, border, tmp.p, h32, v32, s);
        case 4: return sep_u8_dispatch<4>(src, dst, dkx, nx, dky, ny, border, tmp.p, h32, v32, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

template <typename PixT, typename AccT, typename KT, int CH>
static int launch_conv2d(const zb_image* src, zb_image* dst, const KT* d_k, int kh, int kw, int border, cudaStream_t s) {
    const int rows = (int)src->rows, cols = (int)src->cols;
    const dim3 grid = row_grid(div_up((size_t)cols, 32), div_up((size_t)rows, 8));
    conv2d_kernel<PixT, AccT, KT, CH><<<grid, kThreads, (size_t)kh * kw * sizeof(KT), s>>>(
        (const PixT*)src->data, (size_t)src->stride * CH, (PixT*)dst->data, (size_t)dst->stride * CH, rows, cols, d_k, kh, kw, border);
    ZB_LAUNCHED();
    return ZB_OK;
}

int convolve_generic(const zb_image* src_in, zb_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border,
                     cudaStream_t s) {
    const int ch = channels_of(pixfmt);
    const size_t size = (size_t)kh * kw;
    if (size > (size_t)kMaxTaps2D) return ZB_ERR_UNSUPPORTED;
    if (pixfmt == ZB_PIX_RGBAF32) return ZB_ERR_UNSUPPORTED;  // convolution.zig:295: struct fields must be u8
    Scratch taps, alias;
    int rc;
    if ((rc = taps.alloc(size * 4, s))) return rc;
    zb_image src = *src_in;
    if (src.data == dst->data) {  // the reference requires disjoint buffers (image.zig:11-15); be safe: snapshot the input
        const size_t pb = pixel_bytes(pixfmt);
        if ((rc = alias.alloc((size_t)src.rows * src.cols * pb, s))) return rc;
        ZB_CUDA(cudaMemcpy2DAsync(alias.p, (size_t)src.cols * pb, src.data, src.stride * pb, (size_t)src.cols * pb, src.rows,
                                  cudaMemcpyDeviceToDevice, s));
        src.data = alias.p;
        src.stride = src.cols;
    }
    if (pixfmt == ZB_PIX_F32) {
        ZB_CUDA(cudaMemcpyAsync(taps.p, kernel, size * 4, cudaMemcpyHostToDevice, s));
        t_last_kernel = "conv2d_generic_f32";
        return launch_conv2d<float, float, float, 1>(&src, dst, (const float*)taps.p, kh, kw, border, s);
    }
    int32_t ki[kMaxTaps2D];
    int64_t sa = 0;
    for (size_t i = 0; i < size; ++i) { ki[i] = (int32_t)roundf(kernel[i] * 256.0f); sa += llabs((long long)ki[i]); }  // :94-111
    const bool a32 = sa * 255 < 2147483647LL - 128;
    if (a32 && !g_force_generic.load()) {   // kernels up to 7 x 7: shared-memory tiles, every source byte extracted once
        rc = convolve_tile_u8(&src, dst, ch, ki, kh, kw, border, s);
        if (rc != ZB_ERR_UNSUPPORTED) return rc;
    }
    ZB_CUDA(cudaMemcpyAsync(taps.p, ki, size * 4, cudaMemcpyHostToDevice, s));
    const int32_t* dk = (const int32_t*)taps.p;
    t_last_kernel = "conv2d_generic_u8";
    switch (ch) {
        case 1: return a32 ? launch_conv2d<uint8_t, int32_t, int32_t, 1>(&src, dst, dk, kh, kw, border, s)
                           : launch_conv2d<uint8_t, long long, int32_t, 1>(&src, dst, dk, kh, kw, border, s);
        case 3: return a32 ? launch_conv2d<uint8_t, int32_t, int32_t, 3>(&src, dst, dk, kh, kw, border, s)
                           : launch_conv2d<uint8_t, long long, int32_t, 3>(&src, dst, dk, kh, kw, border, s);
        case 4: return a32 ? launch_conv2d<uint8_t, int32_t, int32_t, 4>(&src, dst, dk, kh, kw, border, s)
                           : launch_conv2d<uint8_t, long long, int32_t, 4>(&src, dst, dk, kh, kw, border, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

}  // namespace zb
