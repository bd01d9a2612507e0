// zb_order.cu -- order-statistic filters (SURVEY 8(f).3): Image.medianBlur / percentileBlur / minBlur / maxBlur / midpointBlur /
// alphaTrimmedMeanBlur (reference image.zig:650-790 -> image/order_statistic_blur.zig:22-413, image/histogram.zig:586-612).
//
// The reference slides a 256-bin histogram over each row (O(256) per pixel and per channel, strictly sequential along the row).
// The value it returns depends only on the multiset of the (2r+1)^2 border-resolved window samples (out-of-range under .zero
// counts as the value 0, :338-347), so the device evaluates each pixel independently from a shared-memory tile:
//   percentile   the smallest v with #{x <= v} > rank: an 8-step bisection over v, each step one pass over the window (radius 1-3: the
//                window lives in registers and the passes are unrolled compare-and-add chains)
//                (rank 0 / area-1, i.e. minBlur / maxBlur, is a single min / max pass);
//   midpoint     (min + max + 1) / 2 from one pass;
//   alpha-trim   two bisections give the t-th smallest and t-th largest value, one more pass the sums below / above them; the
//                trimmed sums follow by counting how many copies of the boundary values the reference's bin walk takes (:377-400).
// Integer arithmetic throughout: results are bit-identical to the histogram walk.  Channels of interleaved pixels are filtered
// independently, exactly as the reference's split / merge does (:199-229).
#include <cmath>

#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {
namespace {

constexpr int kTileW = 32, kTileH = 8;
constexpr int kMaxRadius = 31;   // up to here the tile fits the default 48 KB of shared memory; larger radii opt in to the SM's full carve-out

enum { MODE_PERCENTILE = 0, MODE_MIDPOINT = 1, MODE_ALPHA = 2 };

struct OrderParams {
    const uint8_t* src;
    uint8_t* dst;
    size_t src_stride, dst_stride;   // pixels
    int rows, cols, radius, border;
    int rank;        // percentile: 0-based rank of the element returned
    int trim_each;   // alpha-trimmed: elements dropped at each end
};

// RADIUS > 0: the window size is a compile-time constant, so the (2r+1)^2 samples of a channel are loaded into registers once and every
// counting pass is a fully unrolled compare-and-add chain; RADIUS == 0: any radius up to kMaxRadius, passes re-read the shared tile.
template <int CH, int MODE, int RADIUS>
__global__ void __launch_bounds__(kTileW* kTileH) order_kernel(const OrderParams p) {
    extern __shared__ uint8_t tile[];
    const int R = RADIUS > 0 ? RADIUS : p.radius, win = 2 * R + 1, area = win * win;
    const int tw = kTileW + 2 * R, th = kTileH + 2 * R;
    const int pitch = (tw * CH + 3) & ~3;
    const int ty = ZB_GRID_ROW();
    if (ty * kTileH >= p.rows) return;   // past the last tile (uniform per block)
    const int row0 = ty * kTileH - R, col0 = blockIdx.x * kTileW - R;
    const int tid = threadIdx.y * kTileW + threadIdx.x;
    for (int i = tid; i < th * tw; i += kTileW * kTileH) {
        const int y = i / tw, x = i - y * tw;
        const int gr = resolve_index(row0 + y, p.rows, p.border), gc = resolve_index(col0 + x, p.cols, p.border);
#pragma unroll
        for (int k = 0; k < CH; ++k)
            tile[y * pitch + x * CH + k] = (gr >= 0 && gc >= 0) ? p.src[((size_t)gr * p.src_stride + gc) * CH + k] : (uint8_t)0;   // getPixel, :338-347
    }
    __syncthreads();
    const int r = ty * kTileH + threadIdx.y, c = blockIdx.x * kTileW + threadIdx.x;
    if (r >= p.rows || c >= p.cols) return;
#pragma unroll
    for (int k = 0; k < CH; ++k) {
        const uint8_t* w0 = tile + threadIdx.y * pitch + threadIdx.x * CH + k;
        constexpr int kRegs = RADIUS > 0 ? (2 * RADIUS + 1) * (2 * RADIUS + 1) : 1;
        int regs[kRegs];
        if constexpr (RADIUS > 0) {
#pragma unroll
            for (int dy = 0; dy < 2 * RADIUS + 1; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2 * RADIUS + 1; ++dx) regs[dy * (2 * RADIUS + 1) + dx] = w0[dy * pitch + dx * CH];
        }
        auto visit = [&](auto&& f) {           // f(sample) for every sample of the window
            if constexpr (RADIUS > 0) {
#pragma unroll
                for (int i = 0; i < kRegs; ++i) f(regs[i]);
            } else {
                for (int dy = 0; dy < win; ++dy) {
                    const uint8_t* row = w0 + dy * pitch;
                    for (int dx = 0; dx < win; ++dx) f((int)row[dx * CH]);
                }
            }
        };
        auto select = [&](int rank) {          // smallest v whose cumulative count exceeds rank (histogram.zig:603-610)
            int lo = 0, hi = 255;
#pragma unroll 1
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                int n = 0;
                visit([&](int x) { n += x <= mid; });
                if (n > rank) hi = mid; else lo = mid + 1;
            }
            return lo;
        };
        int mn = 255, mx = 0;
        if (MODE == MODE_MIDPOINT || (MODE == MODE_PERCENTILE && (p.rank == 0 || p.rank == area - 1)))
            visit([&](int x) { mn = min(mn, x); mx = max(mx, x); });
        int result;
        if (MODE == MODE_MIDPOINT) {
            result = (mn + mx + 1) >> 1;                                       // :357-365
        } else if (MODE == MODE_PERCENTILE) {
            result = p.rank == 0 ? mn : (p.rank == area - 1 ? mx : select(p.rank));
        } else {
            const int t = p.trim_each;
            const int kept = area - 2 * t;                                     // low_count == high_count == t (the window always holds `area` samples)
            int v_lo = 0, v_hi = 255;
            if (t > 0) {
                v_lo = select(t - 1);          // the t-th smallest sample
                v_hi = select(area - t);       // the t-th largest sample
            }
            unsigned total = 0, sum_lt = 0, sum_gt = 0;
            int cnt_lt = 0, cnt_gt = 0;
            visit([&](int x) {
                total += x;
                if (x < v_lo) { sum_lt += x; ++cnt_lt; }
                if (x > v_hi) { sum_gt += x; ++cnt_gt; }
            });
            unsigned kept_sum = total;
            if (t > 0) kept_sum -= sum_lt + (unsigned)(t - cnt_lt) * v_lo + sum_gt + (unsigned)(t - cnt_gt) * v_hi;   // :377-400
            const unsigned rounded = (kept_sum + (unsigned)kept / 2) / (unsigned)kept;                                 // :405
            result = (int)min(rounded, 255u);
        }
        p.dst[((size_t)r * p.dst_stride + c) * CH + k] = (uint8_t)result;
    }
}

template <int CH, int MODE, int RADIUS>
int launch_kernel(const OrderParams& p, dim3 grid, dim3 block, size_t smem, cudaStream_t s) {
    if (smem > 48 * 1024) ZB_CUDA(cudaFuncSetAttribute(order_kernel<CH, MODE, RADIUS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    order_kernel<CH, MODE, RADIUS><<<grid, block, smem, s>>>(p);
    return ZB_OK;
}
template <int CH, int RADIUS>
int launch_radius(const OrderParams& p, int mode, dim3 grid, dim3 block, size_t smem, cudaStream_t s) {
    int rc;
    switch (mode) {
        case MODE_PERCENTILE: rc = launch_kernel<CH, MODE_PERCENTILE, RADIUS>(p, grid, block, smem, s); break;
        case MODE_MIDPOINT: rc = launch_kernel<CH, MODE_MIDPOINT, RADIUS>(p, grid, block, smem, s); break;
        default: rc = launch_kernel<CH, MODE_ALPHA, RADIUS>(p, grid, block, smem, s); break;
    }
    if (rc) return rc;
    ZB_LAUNCHED();
    return ZB_OK;
}

template <int CH>
int launch_mode(const OrderParams& p, int mode, cudaStream_t s) {
    const int tw = kTileW + 2 * p.radius, th = kTileH + 2 * p.radius;
    const size_t smem = (size_t)th * ((tw * CH + 3) & ~3);
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (smem > di.smem_optin) return ZB_ERR_UNSUPPORTED;   // radius beyond ~100 (Rgba) / ~220 (gray): the window no longer fits one SM
    const dim3 grid = row_grid(div_up(p.cols, kTileW), div_up(p.rows, kTileH)), block(kTileW, kTileH);
    switch (g_force_generic.load() ? 0 : p.radius) {     // zb_set_force_generic: the any-radius kernel, as the cross-check of the unrolled ones
        case 1: return launch_radius<CH, 1>(p, mode, grid, block, smem, s);
        case 2: return launch_radius<CH, 2>(p, mode, grid, block, smem, s);
        case 3: return launch_radius<CH, 3>(p, mode, grid, block, smem, s);
        default: return launch_radius<CH, 0>(p, mode, grid, block, smem, s);
    }
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_order_blur(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, int mode, double param, int border,
                             zb_stream stream) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (mode != ZB_ORDER_PERCENTILE && mode != ZB_ORDER_MIDPOINT && mode != ZB_ORDER_ALPHA_TRIMMED) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;      // image.zig:679 hasSameShape
    if (src->rows == 0 || src->cols == 0) return ZB_OK;                                          // order_statistic_blur.zig:39,111,156
    if (mode == ZB_ORDER_ALPHA_TRIMMED && (!std::isfinite(param) || param < 0.0 || param >= 0.5)) return ZB_ERR_INVALID_TRIM;   // :160
    cudaStream_t s = (cudaStream_t)stream;
    if (radius == 0) return zb_copy(src, dst, pixfmt, stream);                                   // :43-46 image.copy(out)
    if (exceeds_int_index(src, pixfmt) || exceeds_int_index(dst, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (mode == ZB_ORDER_PERCENTILE && !(param >= 0.0 && param <= 1.0)) return ZB_ERR_INVALID_PERCENTILE;   // :48-50 (NaN trips the reference's assert)
    if (!pixfmt_in(kFmt8Bit, pixfmt)) return ZB_ERR_UNSUPPORTED;  // :66,74 UnsupportedPixelType
    if (radius > 4096) return ZB_ERR_UNSUPPORTED;   // (the shared-memory check in launch_mode is the real limit)
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const int ch = channels_of(pixfmt);
    const size_t area = (size_t)(2 * radius + 1) * (2 * radius + 1);
    OrderParams p{};
    p.src = (const uint8_t*)src->data;
    p.dst = (uint8_t*)dst->data;
    p.src_stride = src->stride;
    p.dst_stride = dst->stride;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.radius = (int)radius;
    p.border = border;
    if (mode == ZB_ORDER_PERCENTILE) {                                                           // histogram.zig:596-600
        const double rank_floor = std::floor(param * (double)(area - 1) + 1e-12);
        size_t rank = (size_t)std::trunc(rank_floor);
        p.rank = (int)(rank > area - 1 ? area - 1 : rank);
    } else if (mode == ZB_ORDER_ALPHA_TRIMMED) {                                                 // order_statistic_blur.zig:370-373
        const size_t trimmed_each = (size_t)std::trunc(std::floor(param * (double)area));
        p.trim_each = (int)(trimmed_each < area / 2 ? trimmed_each : area / 2);
    }
    // Every block reads a halo that other blocks write when the images alias (:52-60 uses a temporary for the same reason).
    Scratch tmp;
    zb_image staged = *dst;
    const bool alias = images_overlap(src, dst, (size_t)ch);
    if (alias) {
        if ((rc = tmp.alloc((size_t)p.rows * p.cols * ch, s))) return rc;
        staged.data = tmp.p;
        staged.stride = src->cols;
        p.dst = (uint8_t*)tmp.p;
        p.dst_stride = src->cols;
    }
    rc = dispatch_pixfmt<kFmt8Bit>(pixfmt, [&](auto f) -> int { return launch_mode<Fmt<decltype(f)::value>::N>(p, mode, s); });
    if (rc) return rc;
    if (alias && (rc = zb_copy(&staged, dst, pixfmt, stream))) return rc;
    t_last_kernel = "order_statistic";
    return ZB_OK;
}
