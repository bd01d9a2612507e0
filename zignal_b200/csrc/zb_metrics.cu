// zb_metrics.cu -- Image.psnr / ssim / meanPixelError (SURVEY 8(f).3; reference image.zig:1105-1147 -> image/metrics.zig:10-251).
//
// The reference reduces in f64 over the whole image on one thread.  On the device:
//   psnr / meanPixelError   one pass over both images; 8-bit formats accumulate the squared / absolute differences as integers
//                           (exact, so the f64 the reference builds from them is reproduced bit for bit), float formats as f64 per
//                           thread; per-block partials are summed on the host in block order, so a result is reproducible.
//   ssim                    every interior pixel evaluates the reference's 11x11 Gaussian-window statistics (:76-104) from a shared
//                           tile of the per-pixel scalars (getPixelScalar, :187-222), with the reference's operation order and no
//                           contraction; only the final sum over pixels is associated differently (blocks, then the host).
// All three return a double to the host, so they wait for the stream.
#include <cmath>
#include <limits>
#include <vector>

#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {
namespace {

constexpr int kDiffBlocksPerSm = 8;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// partial[2 * block] = sum of squared differences, partial[2 * block + 1] = sum of absolute differences over the block's pixels;
// Acc = unsigned long long (8-bit formats) or double (float formats), both 8 bytes.
template <int CH, typename Comp, typename Acc>
__global__ void __launch_bounds__(256) diff_sums_kernel(const Comp* __restrict__ a, size_t a_stride, const Comp* __restrict__ b, size_t b_stride,
                                                        int rows, int cols, Acc* __restrict__ partial) {
    const size_t n = (size_t)rows * cols;
    Acc sq = 0, ab = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / cols, c = i - r * cols;
        const Comp* pa = a + (r * a_stride + c) * CH;
        const Comp* pb = b + (r * b_stride + c) * CH;
#pragma unroll
        for (int k = 0; k < CH; ++k) {
            if constexpr (sizeof(Comp) == 1) {
                const int d = (int)pa[k] - (int)pb[k];
                sq += (Acc)(d * d);
                ab += (Acc)abs(d);
            } else {
                const double d = __dsub_rn((double)pa[k], (double)pb[k]);      // metrics.zig:27,133: as(f64, a) - as(f64, b)
                sq = __dadd_rn(sq, __dmul_rn(d, d));
                ab = __dadd_rn(ab, fabs(d));
            }
        }
    }
    __shared__ Acc red[2][8];
    sq = warp_sum(sq);
    ab = warp_sum(ab);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][warp] = sq; red[1][warp] = ab; }
    __syncthreads();
    if (threadIdx.x == 0) {
        Acc s = 0, t = 0;
        for (int w = 0; w < 8; ++w) { s += red[0][w]; t += red[1][w]; }
        partial[2 * blockIdx.x] = s;
        partial[2 * blockIdx.x + 1] = t;
    }
}

struct SsimWindow { double w[121]; };

// getPixelScalar (metrics.zig:187-222).  PIX: 0 = u8, 1 = f32, 2 = Rgb(u8), 3 = Rgba(u8), 4 = Rgba(f32).
template <int PIX>
__device__ __forceinline__ double pixel_scalar(const void* base, size_t stride, int r, int c) {
    const size_t i = (size_t)r * stride + c;
    if constexpr (PIX == 0) {
        return (double)((const uint8_t*)base)[i];
    } else if constexpr (PIX == 1) {
        return (double)((const float*)base)[i];
    } else if constexpr (PIX == 2 || PIX == 3) {
        constexpr int CH = PIX == 2 ? 3 : 4;
        const uint8_t* px = (const uint8_t*)base + i * CH;
        const double rf = __ddiv_rn((double)px[0], 255.0), gf = __ddiv_rn((double)px[1], 255.0), bf = __ddiv_rn((double)px[2], 255.0);
        const double luma = __dadd_rn(__dadd_rn(__dmul_rn(0.2126, rf), __dmul_rn(0.7152, gf)), __dmul_rn(0.0722, bf));   // color.zig:1021-1027
        return __dmul_rn(luma, 255.0);
    } else {
        const float4 v = *(const float4*)((const float*)base + i * 4);
        double sum = 0.0;
        sum = __dadd_rn(sum, (double)v.x);
        sum = __dadd_rn(sum, (double)v.y);
        sum = __dadd_rn(sum, (double)v.z);
        sum = __dadd_rn(sum, (double)v.w);
        return __ddiv_rn(sum, 4.0);
    }
}

constexpr int kSsimW = 32, kSsimH = 8, kSsimTW = kSsimW + 10, kSsimTH = kSsimH + 10;

template <int PIX>
__global__ void __launch_bounds__(kSsimW* kSsimH) ssim_kernel(const void* __restrict__ a, size_t a_stride, const void* __restrict__ b, size_t b_stride,
                                                              int rows, int cols, double c1, double c2, const SsimWindow win,
                                                              double* __restrict__ partial) {
    __shared__ double tx[kSsimTH][kSsimTW + 1], ty[kSsimTH][kSsimTW + 1];
    const int tile = ZB_GRID_ROW();
    const int r0 = tile * kSsimH, c0 = blockIdx.x * kSsimW;           // tile origin == first window row / column of the block
    if (r0 >= rows - 10) return;                                         // past the last tile (uniform per block)
    const int tid = threadIdx.y * kSsimW + threadIdx.x;
    for (int i = tid; i < kSsimTH * kSsimTW; i += kSsimW * kSsimH) {
        const int y = i / kSsimTW, x = i - y * kSsimTW;
        const int gr = r0 + y, gc = c0 + x;
        const bool in = gr < rows && gc < cols;
        tx[y][x] = in ? pixel_scalar<PIX>(a, a_stride, gr, gc) : 0.0;
        ty[y][x] = in ? pixel_scalar<PIX>(b, b_stride, gr, gc) : 0.0;
    }
    __syncthreads();
    double value = 0.0;
    const int orow = r0 + threadIdx.y, ocol = c0 + threadIdx.x;        // output (window-origin) coordinates; centre = (+5, +5)
    if (orow < rows - 10 && ocol < cols - 10) {
        double mu_x = 0.0, mu_y = 0.0, mu_x_sq = 0.0, mu_y_sq = 0.0, mu_xy = 0.0;
        for (int dy = 0; dy < 11; ++dy)
#pragma unroll
            for (int dx = 0; dx < 11; ++dx) {
                const double w = win.w[dy * 11 + dx];
                const double vx = tx[threadIdx.y + dy][threadIdx.x + dx], vy = ty[threadIdx.y + dy][threadIdx.x + dx];
                const double wx = __dmul_rn(w, vx), wy = __dmul_rn(w, vy);
                mu_x = __dadd_rn(mu_x, wx);                                  // :89-93
                mu_y = __dadd_rn(mu_y, wy);
                mu_x_sq = __dadd_rn(mu_x_sq, __dmul_rn(wx, vx));
                mu_y_sq = __dadd_rn(mu_y_sq, __dmul_rn(wy, vy));
                mu_xy = __dadd_rn(mu_xy, __dmul_rn(wx, vy));
            }
        const double sigma_x_sq = fmax(0.0, __dsub_rn(mu_x_sq, __dmul_rn(mu_x, mu_x)));   // :97-99
        const double sigma_y_sq = fmax(0.0, __dsub_rn(mu_y_sq, __dmul_rn(mu_y, mu_y)));
        const double sigma_xy = __dsub_rn(mu_xy, __dmul_rn(mu_x, mu_y));
        const double numerator = __dmul_rn(__dadd_rn(__dmul_rn(__dmul_rn(2.0, mu_x), mu_y), c1), __dadd_rn(__dmul_rn(2.0, sigma_xy), c2));
        const double denominator =
            __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(mu_x, mu_x), __dmul_rn(mu_y, mu_y)), c1), __dadd_rn(__dadd_rn(sigma_x_sq, sigma_y_sq), c2));
        value = __ddiv_rn(numerator, denominator);
    }
    __shared__ double red[kSsimH];
    value = warp_sum(value);
    if (threadIdx.x == 0) red[threadIdx.y] = value;
    __syncthreads();
    if (tid == 0) {
        double s = 0.0;
        for (int w = 0; w < kSsimH; ++w) s = __dadd_rn(s, red[w]);
        partial[(size_t)tile * gridDim.x + blockIdx.x] = s;   // the linear block index: the host sums in this order
    }
}

inline double component_max(int pixfmt) { return is_float_fmt(pixfmt) ? 1.0 : 255.0; }     // metrics.zig:176-185

// Sum of squared and of absolute component differences, as the f64 values the reference's running sums hold.
int diff_sums(const zb_image* a, const zb_image* b, int pixfmt, double* sum_sq, double* sum_abs, cudaStream_t s) {
    *sum_sq = *sum_abs = 0.0;
    if (a->rows == 0 || a->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const int rows = (int)a->rows, cols = (int)a->cols;
    const size_t n = (size_t)rows * cols;
    const int blocks = (int)std::min<size_t>((size_t)di.sm_count * kDiffBlocksPerSm, (n + 255) / 256);
    Scratch buf;
    if ((rc = buf.alloc((size_t)blocks * 16, s))) return rc;
    const bool flt = is_float_fmt(pixfmt);
    rc = dispatch_pixfmt<kFmtAll>(pixfmt, [&](auto f) -> int {
        using P = Fmt<decltype(f)::value>;
        using CT = typename P::CT;
        using Acc = std::conditional_t<std::is_same_v<CT, float>, double, unsigned long long>;
        diff_sums_kernel<P::N, CT, Acc><<<blocks, 256, 0, s>>>((const CT*)a->data, a->stride, (const CT*)b->data, b->stride, rows, cols,
                                                               buf.as<Acc>());
        ZB_LAUNCHED();
        return ZB_OK;
    });
    if (rc) return rc;
    std::vector<unsigned long long> host((size_t)blocks * 2);
    ZB_CUDA(cudaMemcpyAsync(host.data(), buf.p, host.size() * 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    if (!flt) {
        unsigned long long sq = 0, ab = 0;
        for (int i = 0; i < blocks; ++i) { sq += host[2 * i]; ab += host[2 * i + 1]; }
        *sum_sq = (double)sq;      // exact below 2^53, where the reference's f64 running sum of integers is exact as well
        *sum_abs = (double)ab;
    } else {
        const double* d = (const double*)host.data();
        double sq = 0.0, ab = 0.0;
        for (int i = 0; i < blocks; ++i) { sq += d[2 * i]; ab += d[2 * i + 1]; }
        *sum_sq = sq;
        *sum_abs = ab;
    }
    t_last_kernel = "diff_sums";
    return ZB_OK;
}

int check_pair(const zb_image* a, const zb_image* b, int pixfmt, const double* out) {
    if (!a || !b || !out) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmtAll, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (a->rows != b->rows || a->cols != b->cols) return ZB_ERR_DIMENSION_MISMATCH;     // metrics.zig:11,57,117
    if (exceeds_int_index(a, pixfmt) || exceeds_int_index(b, pixfmt)) return ZB_ERR_UNSUPPORTED;
    return ZB_OK;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_psnr(const zb_image* a, const zb_image* b, int pixfmt, double* out, zb_stream stream) {
    int rc = check_pair(a, b, pixfmt, out);
    if (rc) return rc;
    double sq, ab;
    if ((rc = diff_sums(a, b, pixfmt, &sq, &ab, (cudaStream_t)stream))) return rc;
    const double count = (double)((size_t)a->rows * a->cols * channels_of(pixfmt));
    const double mse = sq / count;                                                        // :49 (0 / 0 = NaN for an empty image, as in Zig)
    if (mse == 0.0) { *out = std::numeric_limits<double>::infinity(); return ZB_OK; }     // :50
    *out = 20.0 * std::log10(component_max(pixfmt)) - 10.0 * std::log10(mse);             // :54
    return ZB_OK;
}

extern "C" int zb_mean_pixel_error(const zb_image* a, const zb_image* b, int pixfmt, double* out, zb_stream stream) {
    int rc = check_pair(a, b, pixfmt, out);
    if (rc) return rc;
    double sq, ab;
    if ((rc = diff_sums(a, b, pixfmt, &sq, &ab, (cudaStream_t)stream))) return rc;
    const size_t count = (size_t)a->rows * a->cols * channels_of(pixfmt);
    if (count == 0) { *out = 0.0; return ZB_OK; }                                         // :159
    *out = (ab / (double)count) / component_max(pixfmt);                                  // :160-165
    return ZB_OK;
}

extern "C" int zb_ssim(const zb_image* a, const zb_image* b, int pixfmt, double* out, zb_stream stream) {
    int rc = check_pair(a, b, pixfmt, out);
    if (rc) return rc;
    if (a->rows < 11 || a->cols < 11) return ZB_ERR_IMAGE_TOO_SMALL;                      // :60-62
    cudaStream_t s = (cudaStream_t)stream;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;
    const int rows = (int)a->rows, cols = (int)a->cols;
    const double l = component_max(pixfmt);
    const double c1 = (0.01 * l) * (0.01 * l), c2 = (0.03 * l) * (0.03 * l);              // :64-68
    SsimWindow win;                                                                        // generateSsimWindow, :232-251
    {
        const double sigma = 1.5;
        double sum = 0.0;
        for (int dy = 0; dy < 11; ++dy)
            for (int dx = 0; dx < 11; ++dx) {
                const double y = (double)dy - 5.0, x = (double)dx - 5.0;
                const double g = std::exp(-(x * x + y * y) / (2.0 * sigma * sigma));
                win.w[dy * 11 + dx] = g;
                sum += g;
            }
        for (double& w : win.w) w /= sum;
    }
    const size_t n_tiles = div_up(rows - 10, kSsimH);
    const dim3 grid = row_grid(div_up(cols - 10, kSsimW), n_tiles), block(kSsimW, kSsimH);
    const size_t blocks = (size_t)grid.x * n_tiles;
    Scratch buf;
    if ((rc = buf.alloc(blocks * sizeof(double), s))) return rc;
    double* partial = buf.as<double>();
    rc = dispatch_pixfmt<kFmtAll>(pixfmt, [&](auto f) -> int {
        ssim_kernel<decltype(f)::value><<<grid, block, 0, s>>>(a->data, a->stride, b->data, b->stride, rows, cols, c1, c2, win, partial);
        ZB_LAUNCHED();
        return ZB_OK;
    });
    if (rc) return rc;
    std::vector<double> host(blocks);
    ZB_CUDA(cudaMemcpyAsync(host.data(), partial, blocks * sizeof(double), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    double ssim_sum = 0.0;
    for (double v : host) ssim_sum += v;
    const double weight_sum = (double)(rows - 10) * (double)(cols - 10);                   // :105 (one per interior pixel)
    *out = ssim_sum / weight_sum;                                                          // :113
    t_last_kernel = "ssim";
    return ZB_OK;
}
