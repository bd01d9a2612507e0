// zb_edges.cu -- Image.sobel (reference image.zig:999-1009 -> edges.zig:33-73), a composition of the hot path (SURVEY 8(f).1):
// gray f32 plane (as(f32, convertColor(u8, px)), color.zig:1031-1041 for the luma; float scalars pass through), two dense 3x3
// convolutions with .replicate through zb_convolve's f32 kernel (the reference's accumulation order), and the magnitude
// sqrt(gx^2 + gy^2) / 4 truncated into a u8 image.  Everything stays on the device; three scratch planes from the pool.
#include <algorithm>
#include <cmath>
#include <vector>

#include "zb_conv.h"
#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {

int gaussian_taps_host(float sigma, std::vector<float>& taps);   // zb_api_conv.cu (image.zig:972-990; edges.zig:663-681 is the same formula)

namespace {

template <int CH, bool IS_FLOAT>
__global__ void __launch_bounds__(256) to_gray_f32_kernel(const void* __restrict__ src, size_t src_stride, float* __restrict__ gray, int rows,
                                                          int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = ZB_GRID_ROW();
    if (c >= cols || r >= rows) return;
    float v;
    if constexpr (IS_FLOAT) {
        v = ((const float*)src)[(size_t)r * src_stride + c];
    } else if constexpr (CH == 1) {
        v = (float)((const uint8_t*)src)[(size_t)r * src_stride + c];
    } else {
        const uint8_t* px = (const uint8_t*)src + ((size_t)r * src_stride + c) * CH;
        const int y = (13933 * (int)px[0] + 46871 * (int)px[1] + 4732 * (int)px[2] + 32768) >> 16;   // rgbToGray(u8)
        v = (float)min(max(y, 0), 255);
    }
    gray[(size_t)r * cols + c] = v;
}

__global__ void __launch_bounds__(256) sobel_magnitude_kernel(const float* __restrict__ gx, const float* __restrict__ gy, uint8_t* __restrict__ dst,
                                                              size_t dst_stride, int rows, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = ZB_GRID_ROW();
    if (c >= cols || r >= rows) return;
    const float a = gx[(size_t)r * cols + c], b = gy[(size_t)r * cols + c];
    const float magnitude = __fsqrt_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)));   // edges.zig:65
    const float scaled = __fdiv_rn(magnitude, 4.0f);                                        // :68
    dst[(size_t)r * dst_stride + c] = (uint8_t)truncf(fmaxf(0.0f, fminf(255.0f, scaled))); // :69
}

// The whole of edges.zig:33-73 in one pass over the image: 9 border-replicated luma samples, both 3x3 correlations with the dense
// convolution's accumulation (acc = acc + px*k, separately rounded, taps in row-major order, zero taps included), magnitude.
// Reads the source once and writes one byte per pixel; values are identical to the composition above by construction.
template <int CH, bool IS_FLOAT>
__global__ void __launch_bounds__(256) sobel_fused_kernel(const void* __restrict__ src, size_t src_stride, uint8_t* __restrict__ dst,
                                                          size_t dst_stride, int rows, int cols) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int r = ZB_GRID_ROW() * 8 + (threadIdx.x >> 5);
    if (c >= cols || r >= rows) return;
    auto luma = [&](int y, int x) -> float {
        y = min(max(y, 0), rows - 1);   // .replicate
        x = min(max(x, 0), cols - 1);
        if constexpr (IS_FLOAT) {
            return ((const float*)src)[(size_t)y * src_stride + x];
        } else if constexpr (CH == 1) {
            return (float)((const uint8_t*)src)[(size_t)y * src_stride + x];
        } else {
            const uint8_t* px = (const uint8_t*)src + ((size_t)y * src_stride + x) * CH;
            const int v = (13933 * (int)px[0] + 46871 * (int)px[1] + 4732 * (int)px[2] + 32768) >> 16;   // rgbToGray(u8)
            return (float)min(max(v, 0), 255);
        }
    };
    const float kx[9] = {-1, 0, 1, -2, 0, 2, -1, 0, 1};   // edges.zig:14-18
    const float ky[9] = {-1, -2, -1, 0, 0, 0, 1, 2, 1};   // :21-25
    float gx = 0.0f, gy = 0.0f;
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float v = luma(r + j - 1, c + i - 1);
            gx = mul_add_unfused(v, kx[3 * j + i], gx);
            gy = mul_add_unfused(v, ky[3 * j + i], gy);
        }
    const float magnitude = __fsqrt_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));
    const float scaled = __fdiv_rn(magnitude, 4.0f);
    dst[(size_t)r * dst_stride + c] = (uint8_t)truncf(fmaxf(0.0f, fminf(255.0f, scaled)));
}

// ---- Canny (edges.zig:212-274) ----------------------------------------------------------------------------------------------------

// as(f32, convertColor(u8, v)) for a float scalar: round(clamp(v, 0, 1) * 255) evaluated in f64 (color.zig:114-118).
__global__ void __launch_bounds__(256) canny_quantize_f32_kernel(const float* __restrict__ src, size_t src_stride, float* __restrict__ gray,
                                                                 int rows, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = ZB_GRID_ROW();
    if (c >= cols || r >= rows) return;
    double d = (double)src[(size_t)r * src_stride + c];
    d = d < 0.0 ? 0.0 : (d > 1.0 ? 1.0 : d);
    gray[(size_t)r * cols + c] = (float)(uint8_t)round(d * 255.0);
}

__global__ void __launch_bounds__(256) canny_magnitude_kernel(const float* __restrict__ gx, const float* __restrict__ gy, float* __restrict__ mag,
                                                              size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float a = gx[i], b = gy[i];
    mag[i] = __fsqrt_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)));   // edges.zig:263
}

// Non-maximum suppression along the quantised gradient direction (edges.zig:691-763) fused with the double threshold of
// applyHysteresis' first pass (:540-547): dst = 255 for a surviving pixel with magnitude >= high (a seed), 1 for a surviving
// pixel with magnitude >= low (a candidate), 0 otherwise.  The outermost ring of pixels is never marked (:713).
constexpr uint8_t kWeak = 1, kEdge = 255;
__global__ void __launch_bounds__(256) canny_nms_kernel(const float* __restrict__ gx, const float* __restrict__ gy, const float* __restrict__ mag,
                                                        uint8_t* __restrict__ dst, size_t dst_stride, int rows, int cols, float low, float high) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int r = ZB_GRID_ROW() * 8 + (threadIdx.x >> 5);
    if (c >= cols || r >= rows) return;
    uint8_t v = 0;
    if (r >= 1 && c >= 1 && r + 1 < rows && c + 1 < cols) {
        const size_t i = (size_t)r * cols + c;
        const float vx = gx[i], vy = gy[i];
        const float ax = fabsf(vx), ay = fabsf(vy);
        const float K = 0.414213562f;   // tan(22.5 deg), :709
        int dr, dc;                     // first neighbour; the second is the opposite one
        if (ay <= __fmul_rn(K, ax)) { dr = 0; dc = -1; }
        else if (ax <= __fmul_rn(K, ay)) { dr = -1; dc = 0; }
        else if (__fmul_rn(vx, vy) > 0.0f) { dr = -1; dc = 1; }
        else { dr = -1; dc = -1; }
        const float m = mag[i];
        const float n1 = mag[(size_t)(r + dr) * cols + (c + dc)];
        const float n2 = mag[(size_t)(r - dr) * cols + (c - dc)];
        if (m >= n1 && m >= n2) v = m >= high ? kEdge : (m >= low ? kWeak : (uint8_t)0);
    }
    dst[(size_t)r * dst_stride + c] = v;
}

// Hysteresis (edges.zig:549-575).  The reference grows the edge set breadth-first from the seeds through 8-connected candidates; the
// result is the closure "candidate connected to a seed through candidates", which does not depend on the visiting order.  Each
// block relaxes a 64x64 tile (plus a one-pixel ring read from its neighbours) to its local fixed point in shared memory; the
// host repeats the pass until no block promoted a pixel.  Promotions are monotone (1 -> 255), so a ring value read while the
// neighbouring block is still writing is merely early or late, and a late one is caught by the next pass.
constexpr int kHystTile = 64;
__global__ void __launch_bounds__(1024) canny_hysteresis_kernel(uint8_t* img, size_t stride, int rows, int cols, int* __restrict__ promoted) {
    __shared__ uint8_t t[kHystTile + 2][kHystTile + 4];
    if (ZB_GRID_ROW() * kHystTile >= rows) return;   // past the last tile (uniform per block)
    const int r0 = ZB_GRID_ROW() * kHystTile - 1, c0 = blockIdx.x * kHystTile - 1;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    int weak_here = 0;
    for (int i = tid; i < (kHystTile + 2) * (kHystTile + 2); i += 1024) {
        const int y = i / (kHystTile + 2), x = i - y * (kHystTile + 2);
        const int gr = r0 + y, gc = c0 + x;
        uint8_t v = 0;
        if (gr >= 0 && gr < rows && gc >= 0 && gc < cols) v = ((const volatile uint8_t*)img)[(size_t)gr * stride + gc];
        t[y][x] = v;
        weak_here |= (v == kWeak);
    }
    if (!__syncthreads_or(weak_here)) return;     // nothing left to decide in this tile
    int any = 0, changed;
    do {
        changed = 0;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const int y = 1 + 2 * threadIdx.y + dy, x = 1 + 2 * threadIdx.x + dx;
                if (t[y][x] != kWeak) continue;
                const bool nb = t[y - 1][x - 1] == kEdge || t[y - 1][x] == kEdge || t[y - 1][x + 1] == kEdge || t[y][x - 1] == kEdge ||
                                t[y][x + 1] == kEdge || t[y + 1][x - 1] == kEdge || t[y + 1][x] == kEdge || t[y + 1][x + 1] == kEdge;
                if (nb) { t[y][x] = kEdge; changed = 1; }
            }
        changed = __syncthreads_or(changed);
        any |= changed;
    } while (changed);
    if (!any) return;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const int y = 1 + 2 * threadIdx.y + dy, x = 1 + 2 * threadIdx.x + dx;
            const int gr = r0 + y, gc = c0 + x;
            if (gr < rows && gc < cols && t[y][x] == kEdge) img[(size_t)gr * stride + gc] = kEdge;
        }
    if (tid == 0) *promoted = 1;
}

// Candidates that were never reached stay 0 in the reference's output.
__global__ void __launch_bounds__(256) canny_finalize_kernel(uint8_t* __restrict__ img, size_t stride, int rows, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = ZB_GRID_ROW();
    if (c >= cols || r >= rows) return;
    uint8_t* p = img + (size_t)r * stride + c;
    if (*p == kWeak) *p = 0;
}

// ---- Shen-Castan (edges.zig:83-198, 283-656) ----------------------------------------------------------------------------------------
//
// The ISEF recurrences (:283-306) are sequential in f32 with every product and sum rounded on its own, so they are not reassociated
// into a parallel scan: each line is one thread's dependent chain, the parallelism is across lines, and the loads of the next stretch of
// lines are issued before the current stretch's chain runs.

// as(f32, convertColor(u8, px)) of one source pixel: the luma of to_gray_f32_kernel for 8-bit colours, canny_quantize_f32_kernel's
// round(clamp(v, 0, 1) * 255) in f64 for a float scalar (color.zig:114-118, 1031-1041).
template <int CH, bool IS_FLOAT>
__device__ __forceinline__ float sc_gray(const void* __restrict__ src, size_t stride, int r, int c) {
    if constexpr (IS_FLOAT) {
        double d = (double)((const float*)src)[(size_t)r * stride + c];
        d = d < 0.0 ? 0.0 : (d > 1.0 ? 1.0 : d);
        return (float)(uint8_t)round(d * 255.0);
    } else if constexpr (CH == 1) {
        return (float)((const uint8_t*)src)[(size_t)r * stride + c];
    } else {
        const uint8_t* px = (const uint8_t*)src + ((size_t)r * stride + c) * CH;
        const int y = (13933 * (int)px[0] + 46871 * (int)px[1] + 4732 * (int)px[2] + 32768) >> 16;   // rgbToGray(u8)
        return (float)min(max(y, 0), 255);
    }
}

// ISEF along the rows (isefFilter2D's first loop, :318-330), fused with the luma.  One warp per 32 rows, one lane per row; 32-column
// chunks are staged through a padded shared tile so that global loads and stores stay coalesced (the shape of sat_row_pass).  Forward:
// temp[i] = b*x[i] + a*temp[i-1] (temp[0] = b*x[0]: the running value starts at 0 and b*x + (+0) is b*x for x >= 0), stored to `line`;
// backward from the right: y[n-1] = temp[n-1], y[i] = b*temp[i] + a*y[i+1], overwriting temp in place.  The registers v[] hold the next
// chunk, loaded before the current chunk's recurrence runs.
template <int CH, bool IS_FLOAT>
__global__ void __launch_bounds__(32) isef_row_pass(const void* __restrict__ src, size_t src_stride, float* __restrict__ gray,
                                                    float* __restrict__ line, int rows, int cols, float b, float a) {
    __shared__ float tile[32][33];
    const int lane = threadIdx.x;
    const int r0 = blockIdx.x * 32;
    const int nr = min(32, rows - r0);
    float v[32];
    float run = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = (i < nr && lane < cols) ? sc_gray<CH, IS_FLOAT>(src, src_stride, r0 + i, lane) : 0.0f;
    for (int c0 = 0; c0 < cols; c0 += 32) {
        const int c = c0 + lane;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            tile[i][lane] = v[i];
            if (i < nr && c < cols) gray[(size_t)(r0 + i) * cols + c] = v[i];
        }
        __syncwarp();
        if (c0 + 32 < cols) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = (i < nr && c + 32 < cols) ? sc_gray<CH, IS_FLOAT>(src, src_stride, r0 + i, c + 32) : 0.0f;
        }
        if (lane < nr) {
#pragma unroll 8
            for (int j = 0; j < 32; ++j) {   // past the last column the chain runs on zeros that are never stored
                run = __fadd_rn(__fmul_rn(b, tile[lane][j]), __fmul_rn(a, run));
                tile[lane][j] = run;
            }
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 32; ++i)
            if (i < nr && c < cols) line[(size_t)(r0 + i) * cols + c] = tile[i][lane];
        __syncwarp();
    }
    // backward; every element a lane loads here it stored itself in the forward sweep
    const int last0 = (cols - 1) / 32 * 32;
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = (i < nr && last0 + lane < cols) ? line[(size_t)(r0 + i) * cols + last0 + lane] : 0.0f;
    for (int c0 = last0; c0 >= 0; c0 -= 32) {
        const int c = c0 + lane;
#pragma unroll
        for (int i = 0; i < 32; ++i) tile[i][lane] = v[i];
        __syncwarp();
        if (c0 > 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = i < nr ? line[(size_t)(r0 + i) * cols + c - 32] : 0.0f;
        }
        if (lane < nr) {
            const int nc = min(32, cols - c0);
            for (int j = nc - 1; j >= 0; --j) {
                const float t = tile[lane][j];
                run = c0 + j == cols - 1 ? t : __fadd_rn(__fmul_rn(b, t), __fmul_rn(a, run));
                tile[lane][j] = run;
            }
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 32; ++i)
            if (i < nr && c < cols) line[(size_t)(r0 + i) * cols + c] = tile[i][lane];
        __syncwarp();
    }
}

// ISEF down the columns (:332-349) on the row result, one thread per column, in place in `line` (the forward value of row r replaces
// the row pass's value there once it has been read).  The backward sweep forms the binary Laplacian image on the way (:106-122):
// bli = smoothed - gray >= 0 ? 1 : 0; it stores `smoothed` back into `line` only when non-maximum suppression needs it.  K rows of
// loads are in flight while the previous K rows' recurrence runs.
constexpr int kColBatch = 16;
__global__ void __launch_bounds__(128) isef_col_pass(float* __restrict__ line, const float* __restrict__ gray, uint8_t* __restrict__ bli,
                                                     int rows, int cols, float b, float a, int keep_smoothed) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float* p = line + c;
    const size_t pitch = (size_t)cols;
    float cur[kColBatch], nxt[kColBatch];
    float run = 0.0f;
#pragma unroll
    for (int i = 0; i < kColBatch; ++i) cur[i] = i < rows ? p[(size_t)i * pitch] : 0.0f;
    for (int r0 = 0; r0 < rows; r0 += kColBatch) {
        if (r0 + kColBatch < rows) {
#pragma unroll
            for (int i = 0; i < kColBatch; ++i) nxt[i] = r0 + kColBatch + i < rows ? p[(size_t)(r0 + kColBatch + i) * pitch] : 0.0f;
        }
#pragma unroll
        for (int i = 0; i < kColBatch; ++i) {
            if (r0 + i < rows) {
                run = __fadd_rn(__fmul_rn(b, cur[i]), __fmul_rn(a, run));
                p[(size_t)(r0 + i) * pitch] = run;
            }
        }
#pragma unroll
        for (int i = 0; i < kColBatch; ++i) cur[i] = nxt[i];
    }
    float gcur[kColBatch], gnxt[kColBatch];
    const float* g = gray + c;
    uint8_t* m = bli + c;
    // batches of rows top - kColBatch + 1 .. top, walked from the bottom of the image up
#pragma unroll
    for (int i = 0; i < kColBatch; ++i) {
        const int r = rows - 1 - i;
        cur[i] = r >= 0 ? p[(size_t)r * pitch] : 0.0f;
        gcur[i] = r >= 0 ? g[(size_t)r * pitch] : 0.0f;
    }
    for (int top = rows - 1; top >= 0; top -= kColBatch) {
        if (top - kColBatch >= 0) {
#pragma unroll
            for (int i = 0; i < kColBatch; ++i) {
                const int r = top - kColBatch - i;
                nxt[i] = r >= 0 ? p[(size_t)r * pitch] : 0.0f;
                gnxt[i] = r >= 0 ? g[(size_t)r * pitch] : 0.0f;
            }
        }
#pragma unroll
        for (int i = 0; i < kColBatch; ++i) {
            const int r = top - i;
            if (r >= 0) {
                run = r == rows - 1 ? cur[i] : __fadd_rn(__fmul_rn(b, cur[i]), __fmul_rn(a, run));
                m[(size_t)r * pitch] = __fsub_rn(run, gcur[i]) >= 0.0f ? 1 : 0;
                if (keep_smoothed) p[(size_t)r * pitch] = run;
            }
        }
#pragma unroll
        for (int i = 0; i < kColBatch; ++i) {
            cur[i] = nxt[i];
            gcur[i] = gnxt[i];
        }
    }
}

// findZeroCrossings (:356-414) at one pixel: forward mode compares with the E, S, SE and SW neighbours (bounds-checked); otherwise the
// interior pixels are compared with their 4-neighbourhood when the image is at least 3 x 3, and every pixel with its in-bounds
// 4-neighbours below that.
__device__ __forceinline__ bool sc_zero_crossing(const uint8_t* __restrict__ bli, int r, int c, int rows, int cols, bool forward) {
    const size_t i = (size_t)r * cols + c;
    const uint8_t center = bli[i];
    if (forward) {
        if (c + 1 < cols && center != bli[i + 1]) return true;
        if (r + 1 < rows) {
            if (center != bli[i + cols]) return true;
            if (c + 1 < cols && center != bli[i + cols + 1]) return true;
            if (c > 0 && center != bli[i + cols - 1]) return true;
        }
        return false;
    }
    if (rows >= 3 && cols >= 3) {
        if (r == 0 || c == 0 || r == rows - 1 || c == cols - 1) return false;
        return center != bli[i - 1] || center != bli[i + 1] || center != bli[i - cols] || center != bli[i + cols];
    }
    return (c > 0 && center != bli[i - 1]) || (c + 1 < cols && center != bli[i + 1]) || (r > 0 && center != bli[i - cols]) ||
           (r + 1 < rows && center != bli[i + cols]);
}

// Integral.sum (integral.zig:85-90): ((D - left) - top) + corner over rows r1..r2, columns c1..c2 inclusive.
__device__ __forceinline__ float sc_box_sum(const float* __restrict__ sat, int cols, int r1, int c1, int r2, int c2) {
    const float D = sat[(size_t)r2 * cols + c2];
    const float left = c1 > 0 ? sat[(size_t)r2 * cols + (c1 - 1)] : 0.0f;
    const float top = r1 > 0 ? sat[(size_t)(r1 - 1) * cols + c2] : 0.0f;
    const float corner = (r1 > 0 && c1 > 0) ? sat[(size_t)(r1 - 1) * cols + (c1 - 1)] : 0.0f;
    return __fadd_rn(__fsub_rn(__fsub_rn(D, left), top), corner);
}

// Device-side state of one call (zeroed before sc_gradient_kernel).
struct ScState {
    unsigned long long hist[256];   // candidates per rounded gradient
    unsigned int ticket;
    int none;                       // no candidate at all: the output is all zeros (:153-161)
    float t_high, t_low;
    int promoted;                   // hysteresis passes
};

// computeAdaptiveGradients (:417-495) at the candidates, 0 elsewhere, plus the histogram of round(clamp(g, 0, 255)) over the candidates
// (:139-152): per-CTA counts in shared memory, added into u64 global counts.  The last CTA to finish (ticket) turns the histogram into
// t_high / t_low (:153-170) on the device.  CTAs stride over rows; the threads of a CTA over the columns of a row.
__global__ void __launch_bounds__(256) sc_gradient_kernel(const uint8_t* __restrict__ bli, const float* __restrict__ sat3, float* __restrict__ grad,
                                                          ScState* st, int rows, int cols, long long half, int forward, float high_ratio,
                                                          float low_rel) {
    __shared__ unsigned int h[256];
    __shared__ bool is_last;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0u;
    __syncthreads();
    const size_t n = (size_t)rows * cols;
    const float* s_gray = sat3;
    const float* s_mask = sat3 + n;
    const float* s_masked = sat3 + 2 * n;
    for (int r = blockIdx.x; r < rows; r += gridDim.x) {
        const int r1 = (int)max((long long)r - half, 0ll), r2 = (int)min((long long)r + half, (long long)rows - 1);
        for (int c = threadIdx.x; c < cols; c += blockDim.x) {
            float g = 0.0f;
            if (sc_zero_crossing(bli, r, c, rows, cols, forward != 0)) {
                const int c1 = (int)max((long long)c - half, 0ll), c2 = (int)min((long long)c + half, (long long)cols - 1);
                const float area = (float)((long long)(r2 - r1 + 1) * (long long)(c2 - c1 + 1));
                const float count1 = sc_box_sum(s_mask, cols, r1, c1, r2, c2);
                const float count0 = __fsub_rn(area, count1);
                if (count0 > 0.0f && count1 > 0.0f) {
                    const float sum1 = sc_box_sum(s_masked, cols, r1, c1, r2, c2);
                    const float sum_total = sc_box_sum(s_gray, cols, r1, c1, r2, c2);
                    const float sum0 = __fsub_rn(sum_total, sum1);
                    const float mean0 = __fdiv_rn(sum0, count0), mean1 = __fdiv_rn(sum1, count1);
                    g = fabsf(__fsub_rn(mean1, mean0));
                }
                atomicAdd(&h[(int)roundf(fminf(fmaxf(g, 0.0f), 255.0f))], 1u);   // @round: half away from zero
            }
            grad[(size_t)r * cols + c] = g;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        if (h[i]) atomicAdd(&st->hist[i], (unsigned long long)h[i]);
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        is_last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1u;
    }
    __syncthreads();
    if (!is_last) return;
    __shared__ unsigned long long hist[256];
    __threadfence();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = __ldcg(&st->hist[i]);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long total = 0;
        for (int i = 0; i < 256; ++i) total += hist[i];
        if (total == 0) {
            st->none = 1;
        } else {
            const unsigned long long target = (unsigned long long)floorf(__fmul_rn(__ull2float_rn(total), high_ratio));
            unsigned long long cum = 0;
            int idx = 0;
            while (idx < 256 && cum < target) cum += hist[idx++];   // idx ends one past the bin that reached the target
            const float t_high = (float)min(idx, 255);
            st->t_high = t_high;
            st->t_low = __fmul_rn(low_rel, t_high);
        }
    }
}

// The output pass: 255 for a kept candidate with g >= t_high, 1 (kWeak, for canny_hysteresis_kernel) for one with g >= t_low when
// hysteresis is on, 0 otherwise; all 0 when there was no candidate.  With use_nms a candidate is kept when its adaptive gradient is not
// below its two neighbours along the direction of the smoothed image's central differences (nonMaxSuppressEdges, :582-656; the
// outermost ring and images under 3 x 3 keep nothing).
__global__ void __launch_bounds__(256) sc_classify_kernel(const uint8_t* __restrict__ bli, const float* __restrict__ grad,
                                                          const float* __restrict__ smoothed, const ScState* __restrict__ st,
                                                          uint8_t* __restrict__ dst, size_t dst_stride, int rows, int cols, int use_nms,
                                                          int hysteresis) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const int r = ZB_GRID_ROW() * 8 + (threadIdx.x >> 5);
    if (c >= cols || r >= rows) return;
    uint8_t v = 0;
    if (!st->none) {
        const size_t i = (size_t)r * cols + c;
        bool keep;
        if (!use_nms) {
            keep = sc_zero_crossing(bli, r, c, rows, cols, true);
        } else {
            keep = false;
            if (r >= 1 && c >= 1 && r + 1 < rows && c + 1 < cols && sc_zero_crossing(bli, r, c, rows, cols, false)) {
                const float gx = __fmul_rn(0.5f, __fsub_rn(smoothed[i + 1], smoothed[i - 1]));
                const float gy = __fmul_rn(0.5f, __fsub_rn(smoothed[i + cols], smoothed[i - cols]));
                const float ax = fabsf(gx), ay = fabsf(gy);
                const float K = 0.414213562f;   // tan(22.5 deg)
                int dr, dc;                     // first neighbour; the second is the opposite one
                if (ay <= __fmul_rn(K, ax)) { dr = 0; dc = -1; }
                else if (ax <= __fmul_rn(K, ay)) { dr = -1; dc = 0; }
                else if (__fmul_rn(gx, gy) > 0.0f) { dr = -1; dc = 1; }
                else { dr = -1; dc = -1; }
                const float m = grad[i];
                const float n1 = grad[(size_t)(r + dr) * cols + (c + dc)];
                const float n2 = grad[(size_t)(r - dr) * cols + (c - dc)];
                keep = m >= n1 && m >= n2;
            }
        }
        if (keep) {
            const float g = grad[i];
            v = g >= st->t_high ? kEdge : (hysteresis && g >= st->t_low ? kWeak : (uint8_t)0);
        }
    }
    dst[(size_t)r * dst_stride + c] = v;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_canny(const zb_image* src, zb_image* dst, int pixfmt, float sigma, float low_threshold, float high_threshold,
                        zb_stream stream) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (!std::isfinite(sigma) || !std::isfinite(low_threshold) || !std::isfinite(high_threshold)) return ZB_ERR_INVALID_ARGUMENT;   // :221
    if (sigma < 0) return ZB_ERR_INVALID_SIGMA;                                                                                     // :224
    if (low_threshold < 0 || high_threshold < 0 || low_threshold >= high_threshold) return ZB_ERR_INVALID_THRESHOLD;               // :225-226
    if (pixfmt != ZB_PIX_U8 && pixfmt != ZB_PIX_F32 && pixfmt != ZB_PIX_RGB8 && pixfmt != ZB_PIX_RGBA8) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    cudaStream_t s = (cudaStream_t)stream;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const int rows = (int)src->rows, cols = (int)src->cols;
    const size_t n = (size_t)rows * cols, plane = n * sizeof(float);
    const int planes = sigma == 0 ? 4 : 5;
    Scratch buf;
    if ((rc = buf.alloc(planes * plane + 256, s))) return rc;
    float* gray = buf.as<float>();
    float* gx = gray + n;
    float* gy = gx + n;
    float* mag = gy + n;
    float* blurred = sigma == 0 ? gray : mag + n;                      // :241-242 (sigma == 0: no blur)
    int* promoted = (int*)((char*)buf.p + planes * plane);

    const dim3 grid = row_grid(div_up(cols, 256), (size_t)rows);
    switch (pixfmt) {                                                  // :229-236
        case ZB_PIX_F32: canny_quantize_f32_kernel<<<grid, 256, 0, s>>>((const float*)src->data, src->stride, gray, rows, cols); break;
        case ZB_PIX_U8: to_gray_f32_kernel<1, false><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
        case ZB_PIX_RGB8: to_gray_f32_kernel<3, false><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
        default: to_gray_f32_kernel<4, false><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
    }
    ZB_LAUNCHED();
    zb_image g{gray, src->rows, src->cols, src->cols}, b{blurred, src->rows, src->cols, src->cols}, ix{gx, src->rows, src->cols, src->cols},
        iy{gy, src->rows, src->cols, src->cols};
    if (sigma != 0) {                                                  // blurGaussian, :663-687
        std::vector<float> taps;
        if ((rc = gaussian_taps_host(sigma, taps))) return rc;
        if ((int)taps.size() > kMaxTaps) return ZB_ERR_UNSUPPORTED;
        if ((rc = conv_separable_generic(&g, &b, ZB_PIX_F32, taps.data(), (int)taps.size(), taps.data(), (int)taps.size(), ZB_BORDER_REPLICATE, s)))
            return rc;
    }
    static const float sobel_x[9] = {-1, 0, 1, -2, 0, 2, -1, 0, 1};   // edges.zig:14-18
    static const float sobel_y[9] = {-1, -2, -1, 0, 0, 0, 1, 2, 1};   // :21-25
    if ((rc = convolve_generic(&b, &ix, ZB_PIX_F32, sobel_x, 3, 3, ZB_BORDER_REPLICATE, s))) return rc;   // :253
    if ((rc = convolve_generic(&b, &iy, ZB_PIX_F32, sobel_y, 3, 3, ZB_BORDER_REPLICATE, s))) return rc;   // :254
    canny_magnitude_kernel<<<div_up(n, 256), 256, 0, s>>>(gx, gy, mag, n);
    ZB_LAUNCHED();
    uint8_t* out = (uint8_t*)dst->data;
    canny_nms_kernel<<<row_grid(div_up(cols, 32), div_up(rows, 8)), 256, 0, s>>>(gx, gy, mag, out, dst->stride, rows, cols, low_threshold,
                                                                                 high_threshold);
    ZB_LAUNCHED();
    const dim3 hgrid = row_grid(div_up(cols, kHystTile), div_up(rows, kHystTile));
    for (;;) {
        int h = 0;
        if (cudaMemsetAsync(promoted, 0, sizeof(int), s) != cudaSuccess) return ZB_ERR_DEVICE_FAILURE;
        canny_hysteresis_kernel<<<hgrid, dim3(32, 32), 0, s>>>(out, dst->stride, rows, cols, promoted);
        ZB_LAUNCHED();
        if (cudaMemcpyAsync(&h, promoted, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess) return ZB_ERR_DEVICE_FAILURE;
        if (cudaStreamSynchronize(s) != cudaSuccess) return ZB_ERR_DEVICE_FAILURE;
        if (!h) break;
    }
    canny_finalize_kernel<<<grid, 256, 0, s>>>(out, dst->stride, rows, cols);
    ZB_LAUNCHED();
    t_last_kernel = "canny";
    return ZB_OK;
}

extern "C" int zb_shen_castan(const zb_image* src, zb_image* dst, int pixfmt, float smooth, uint64_t window_size, float high_ratio,
                              float low_rel, int hysteresis, int use_nms, zb_stream stream) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (pixfmt != ZB_PIX_U8 && pixfmt != ZB_PIX_F32 && pixfmt != ZB_PIX_RGB8 && pixfmt != ZB_PIX_RGBA8) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;   // image.zig:1023
    if (!(smooth > 0.0f && smooth < 1.0f)) return ZB_ERR_INVALID_B_PARAMETER;                  // ShenCastan.zig:40
    if (window_size % 2 == 0) return ZB_ERR_WINDOW_SIZE_MUST_BE_ODD;                            // :41
    if (window_size < 3) return ZB_ERR_WINDOW_SIZE_TOO_SMALL;                                   // :42
    if (!(high_ratio > 0.0f && high_ratio < 1.0f)) return ZB_ERR_INVALID_THRESHOLD;            // :43
    if (!(low_rel > 0.0f && low_rel < 1.0f)) return ZB_ERR_INVALID_THRESHOLD;                  // :44
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    if (src->cols > 0x7fffffffu) return ZB_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const int rows = (int)src->rows, cols = (int)src->cols;
    const size_t n = (size_t)rows * cols, plane = n * sizeof(float);
    const float b = smooth, a = 1.0f - smooth;                                                  // edges.zig:287
    const long long half = (long long)std::min<uint64_t>(window_size / 2, (uint64_t)1 << 40);   // clipping makes anything larger equivalent
    // scratch: state | gray | line (row result -> column temp -> smoothed) | gradients (own plane only when NMS reads `smoothed`) |
    // three summed-area tables | bli
    const size_t state_bytes = (sizeof(ScState) + 255) / 256 * 256;
    const int fplanes = use_nms ? 6 : 5;
    Scratch buf;
    if ((rc = buf.alloc(state_bytes + fplanes * plane + n, s))) return rc;
    ScState* st = buf.as<ScState>();
    float* gray = (float*)((char*)buf.p + state_bytes);
    float* line = gray + n;
    float* grad = use_nms ? line + n : line;
    float* sat3 = grad + n;
    uint8_t* bli = (uint8_t*)(sat3 + 3 * n);

    const unsigned row_blocks = div_up(rows, 32);
    switch (pixfmt) {                                                                          // :91-100 luma, :318-330 ISEF rows
        case ZB_PIX_F32: isef_row_pass<1, true><<<row_blocks, 32, 0, s>>>(src->data, src->stride, gray, line, rows, cols, b, a); break;
        case ZB_PIX_U8: isef_row_pass<1, false><<<row_blocks, 32, 0, s>>>(src->data, src->stride, gray, line, rows, cols, b, a); break;
        case ZB_PIX_RGB8: isef_row_pass<3, false><<<row_blocks, 32, 0, s>>>(src->data, src->stride, gray, line, rows, cols, b, a); break;
        default: isef_row_pass<4, false><<<row_blocks, 32, 0, s>>>(src->data, src->stride, gray, line, rows, cols, b, a); break;
    }
    ZB_LAUNCHED();
    isef_col_pass<<<div_up(cols, 128), 128, 0, s>>>(line, gray, bli, rows, cols, b, a, use_nms ? 1 : 0);   // :332-349, :106-122
    ZB_LAUNCHED();
    if ((rc = sat_gray_mask(gray, bli, sat3, rows, cols, s))) return rc;                     // :434-452
    ZB_CUDA(cudaMemsetAsync(st, 0, sizeof(ScState), s));
    const unsigned grad_blocks = (unsigned)std::min<size_t>((size_t)rows, (size_t)di.sm_count * 8);
    sc_gradient_kernel<<<grad_blocks, 256, 0, s>>>(bli, sat3, grad, st, rows, cols, half, use_nms ? 0 : 1, high_ratio, low_rel);
    ZB_LAUNCHED();
    uint8_t* out = (uint8_t*)dst->data;                                                       // every source read is done by now
    sc_classify_kernel<<<row_grid(div_up(cols, 32), div_up(rows, 8)), 256, 0, s>>>(bli, grad, line, st, out, dst->stride, rows, cols,
                                                                                   use_nms ? 1 : 0, hysteresis ? 1 : 0);
    ZB_LAUNCHED();
    t_last_kernel = "shen_castan";
    if (!hysteresis) return ZB_OK;                                                             // :183-193
    const dim3 hgrid = row_grid(div_up(cols, kHystTile), div_up(rows, kHystTile));           // applyHysteresis, :499-575
    int* promoted = &st->promoted;
    for (;;) {
        int h = 0;
        if (cudaMemsetAsync(promoted, 0, sizeof(int), s) != cudaSuccess) return ZB_ERR_DEVICE_FAILURE;
        canny_hysteresis_kernel<<<hgrid, dim3(32, 32), 0, s>>>(out, dst->stride, rows, cols, promoted);
        ZB_LAUNCHED();
        if (cudaMemcpyAsync(&h, promoted, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess) return ZB_ERR_DEVICE_FAILURE;
        if (cudaStreamSynchronize(s) != cudaSuccess) return ZB_ERR_DEVICE_FAILURE;
        if (!h) break;
    }
    canny_finalize_kernel<<<row_grid(div_up(cols, 256), (size_t)rows), 256, 0, s>>>(out, dst->stride, rows, cols);
    ZB_LAUNCHED();
    return ZB_OK;
}

extern "C" int zb_sobel(const zb_image* src, zb_image* dst, int pixfmt, zb_stream stream) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (pixfmt != ZB_PIX_U8 && pixfmt != ZB_PIX_F32 && pixfmt != ZB_PIX_RGB8 && pixfmt != ZB_PIX_RGBA8) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;   // image.zig:1005
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    cudaStream_t s = (cudaStream_t)stream;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const int rows = (int)src->rows, cols = (int)src->cols;
    if (!g_force_generic.load()) {   // one pass; the composition below stays as the cross-check (zb_set_force_generic)
        if (pixfmt != ZB_PIX_F32 && g_tune_sobel_tile.load()) {   // 8-bit input: shared-memory byte tiles (luma on the way in), integer gradients (zb_conv_tile_u8.cu)
            rc = sobel_tile_u8(src, dst, channels_of(pixfmt), s);
            if (rc != ZB_ERR_UNSUPPORTED) {
                if (rc == ZB_OK) t_last_kernel = "sobel_tile_u8";
                return rc;
            }
        }
        const dim3 g2 = row_grid(div_up(cols, 32), div_up(rows, 8));
        uint8_t* dp = (uint8_t*)dst->data;
        switch (pixfmt) {
            case ZB_PIX_F32: sobel_fused_kernel<1, true><<<g2, 256, 0, s>>>(src->data, src->stride, dp, dst->stride, rows, cols); break;
            case ZB_PIX_U8: sobel_fused_kernel<1, false><<<g2, 256, 0, s>>>(src->data, src->stride, dp, dst->stride, rows, cols); break;
            case ZB_PIX_RGB8: sobel_fused_kernel<3, false><<<g2, 256, 0, s>>>(src->data, src->stride, dp, dst->stride, rows, cols); break;
            default: sobel_fused_kernel<4, false><<<g2, 256, 0, s>>>(src->data, src->stride, dp, dst->stride, rows, cols); break;
        }
        ZB_LAUNCHED();
        t_last_kernel = "sobel_fused";
        return ZB_OK;
    }
    const size_t plane = (size_t)rows * cols * sizeof(float);
    Scratch buf;
    if ((rc = buf.alloc(3 * plane, s))) return rc;
    float* gray = buf.as<float>();
    float* gx = gray + (size_t)rows * cols;
    float* gy = gx + (size_t)rows * cols;
    const dim3 grid = row_grid(div_up(cols, 256), (size_t)rows);
    switch (pixfmt) {
        case ZB_PIX_F32: to_gray_f32_kernel<1, true><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
        case ZB_PIX_U8: to_gray_f32_kernel<1, false><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
        case ZB_PIX_RGB8: to_gray_f32_kernel<3, false><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
        default: to_gray_f32_kernel<4, false><<<grid, 256, 0, s>>>(src->data, src->stride, gray, rows, cols); break;
    }
    ZB_LAUNCHED();
    static const float sobel_x[9] = {-1, 0, 1, -2, 0, 2, -1, 0, 1};   // edges.zig:14-18
    static const float sobel_y[9] = {-1, -2, -1, 0, 0, 0, 1, 2, 1};   // :21-25
    zb_image g{gray, src->rows, src->cols, src->cols}, ix{gx, src->rows, src->cols, src->cols}, iy{gy, src->rows, src->cols, src->cols};
    if ((rc = convolve_generic(&g, &ix, ZB_PIX_F32, sobel_x, 3, 3, ZB_BORDER_REPLICATE, s))) return rc;
    if ((rc = convolve_generic(&g, &iy, ZB_PIX_F32, sobel_y, 3, 3, ZB_BORDER_REPLICATE, s))) return rc;
    sobel_magnitude_kernel<<<grid, 256, 0, s>>>(gx, gy, (uint8_t*)dst->data, dst->stride, rows, cols);
    ZB_LAUNCHED();
    t_last_kernel = "sobel";
    return ZB_OK;
}
