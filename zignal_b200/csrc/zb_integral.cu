// zb_integral.cu -- Image.integral / boxBlur / sharpen via f32 summed-area tables.
//
// Reference: integral.zig:41-78 (plane), :85-90 (sum), :194-269 (boxBlurPlane), :325-422
// (sharpenPlane), :273-322 (struct sharpen), image.zig:635-648, :785-799.
//
// The SAT is f32 even for u8 input and sums above 2^24 are inexact, so the summation ORDER is part
// of the result (SURVEY appendix A.6).  The kernels keep the reference's order exactly:
//   1. row pass   : sequential f32 running sum along each row (one lane owns one row; a warp stages
//                   32x32 tiles through shared memory so global accesses stay coalesced);
//   2. column pass: sat[r][c] = sat[r-1][c] + sat[r][c], sequential down each column (one thread per
//                   column, coalesced across threads);
//   3. evaluation : ((D - left) - top) + corner, divided by the clipped-window area; windows are
//                   clipped to the image, not padded; ints round half away and saturate.
// All adds/subs/divs use the _rn intrinsics so nothing is contracted or reassociated.
#include "zb_device.cuh"
#include "zb_host_stage.h"
#include "zb_internal.h"

namespace zb {

// zb_box_fused.cu: 8-bit gray / Rgba without the SAT round trip through HBM (bit-identical results)
int box_fused_u8(const zb_image* src, zb_image* dst, int channels, uint32_t radius, int mode, float c, cudaStream_t s);

namespace {

// What the evaluation pass makes of the clipped-window sum.
enum { EVAL_BOX = 0, EVAL_SHARPEN = 1, EVAL_THRESHOLD = 2 };

// ---- 1. row pass -------------------------------------------------------------------------------
// One warp sweeps rows [r0, r0 + 32) of one plane; fetch(r, c) yields the f32 source element.
template <typename Fetch>
__device__ __forceinline__ void sat_row_sweep(Fetch fetch, float* __restrict__ plane, int r0, int rows, int cols) {
    __shared__ float tile[32][33];
    const int lane = threadIdx.x;
    const int nr = min(32, rows - r0);
    float run = 0.0f;  // running sum of row r0 + lane
    for (int c0 = 0; c0 < cols; c0 += 32) {
        const int nc = min(32, cols - c0);
        for (int i = 0; i < nr; ++i)
            tile[i][lane] = lane < nc ? fetch(r0 + i, c0 + lane) : 0.0f;
        __syncwarp();
        if (lane < nr) {
#pragma unroll 8
            for (int j = 0; j < 32; ++j) {  // adding the 0.0f padding of a partial tile changes nothing that is stored
                run = __fadd_rn(run, tile[lane][j]);
                tile[lane][j] = run;
            }
        }
        __syncwarp();
        for (int i = 0; i < nr; ++i)
            if (lane < nc) plane[(size_t)(r0 + i) * cols + c0 + lane] = tile[i][lane];
        __syncwarp();
    }
}

// grid: (ceil(rows/32), CH); block: 32 threads (one warp).  sat plane k is rows x cols contiguous.
template <typename SrcT, int CH>
__global__ void __launch_bounds__(32) sat_row_pass(const SrcT* __restrict__ src, size_t src_row_el, float* __restrict__ sat,
                                                   int rows, int cols) {
    const int k = blockIdx.y;
    sat_row_sweep([&](int r, int c) { return (float)src[(size_t)r * src_row_el + (size_t)c * CH + k]; }, sat + (size_t)k * rows * cols,
                  blockIdx.x * 32, rows, cols);
}

// The three tables of Shen-Castan's adaptive gradient (edges.zig:434-452): plane 0 of gray, plane 1 of the 0 / 1 mask (the u8 path:
// as(f32, v) is exact) and plane 2 of gray[i] * f32(mask[i]).  grid: (ceil(rows/32), 3).
__global__ void __launch_bounds__(32) sat_row_pass_gray_mask(const float* __restrict__ gray, const uint8_t* __restrict__ mask,
                                                             float* __restrict__ sat, int rows, int cols) {
    const int k = blockIdx.y;
    sat_row_sweep(
        [&](int r, int c) {
            const size_t i = (size_t)r * cols + c;
            if (k == 0) return gray[i];
            if (k == 1) return (float)mask[i];
            return __fmul_rn(gray[i], (float)mask[i]);
        },
        sat + (size_t)k * rows * cols, blockIdx.x * 32, rows, cols);
}

// ---- 2. column pass ------------------------------------------------------------------------------
// one thread per (plane, column); rows are walked sequentially.
__global__ void __launch_bounds__(256) sat_col_pass(float* __restrict__ sat, int rows, int cols, int planes) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)planes * cols) return;
    const int k = (int)(idx / cols), c = (int)(idx - (size_t)k * cols);
    float* p = sat + (size_t)k * rows * cols + c;
    float run = p[0];
    int r = 1;
    for (; r + 8 <= rows; r += 8) {
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = p[(size_t)(r + i) * cols];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            run = __fadd_rn(run, v[i]);
            p[(size_t)(r + i) * cols] = run;
        }
    }
    for (; r < rows; ++r) {
        run = __fadd_rn(run, p[(size_t)r * cols]);
        p[(size_t)r * cols] = run;
    }
}

// ---- 3. evaluation -------------------------------------------------------------------------------
// EVAL_THRESHOLD (thresholdAdaptiveMean, binary.zig:86-119; u8 only): dst = f32(src) > fl(fl(S / area) - c) ? 255 : 0.  Each thread
// reads its own source pixel before writing the same pixel of dst, so src may be dst (as for sharpen).
template <typename PixT, int CH, int MODE>
__global__ void __launch_bounds__(256) sat_eval(const float* __restrict__ sat, const PixT* __restrict__ src, size_t src_row_el,
                                                PixT* __restrict__ dst, size_t dst_row_el, int rows, int cols, int radius, float offset) {
    const int r = ZB_GRID_ROW();
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= cols * CH || r >= rows) return;
    const int c = e / CH, k = e - c * CH;
    const float* plane = sat + (size_t)k * rows * cols;
    const int r1 = max(r - radius, 0), r2 = min(r + radius, rows - 1);  // r -| radius ; @min(r + radius, rows - 1)
    const int c1 = max(c - radius, 0), c2 = min(c + radius, cols - 1);
    const float area = (float)((long long)(r2 - r1 + 1) * (long long)(c2 - c1 + 1));
    const float D = plane[(size_t)r2 * cols + c2];
    const float left = c1 > 0 ? plane[(size_t)r2 * cols + (c1 - 1)] : 0.0f;
    const float top = r1 > 0 ? plane[(size_t)(r1 - 1) * cols + c2] : 0.0f;
    const float corner = (r1 > 0 && c1 > 0) ? plane[(size_t)(r1 - 1) * cols + (c1 - 1)] : 0.0f;
    const float s = __fadd_rn(__fsub_rn(__fsub_rn(D, left), top), corner);  // integral.zig:86-89
    float val = __fdiv_rn(s, area);
    if constexpr (MODE == EVAL_THRESHOLD) {
        const float original = (float)src[(size_t)r * src_row_el + e];
        dst[(size_t)r * dst_row_el + e] = original > __fsub_rn(val, offset) ? (PixT)255 : (PixT)0;
        return;
    }
    if constexpr (MODE == EVAL_SHARPEN) {
        const float original = (float)src[(size_t)r * src_row_el + e];
        val = __fsub_rn(__fmul_rn(2.0f, original), val);  // integral.zig:357 / :310
    }
    if constexpr (sizeof(PixT) == 1) dst[(size_t)r * dst_row_el + e] = clamp_u8_from_float(val);
    else dst[(size_t)r * dst_row_el + e] = val;
}

template <typename SrcT, int CH>
int build_sat(const zb_image* src, float* sat, cudaStream_t s) {
    const int rows = (int)src->rows, cols = (int)src->cols;
    dim3 grid(div_up(rows, 32), CH);
    sat_row_pass<SrcT, CH><<<grid, 32, 0, s>>>((const SrcT*)src->data, (size_t)src->stride * CH, sat, rows, cols);
    ZB_LAUNCHED();
    sat_col_pass<<<div_up((size_t)cols * CH, 256), 256, 0, s>>>(sat, rows, cols, CH);
    ZB_LAUNCHED();
    return ZB_OK;
}

template <typename PixT, int CH, int MODE>
int box_or_sharpen(const zb_image* src, zb_image* dst, int radius, float c, cudaStream_t s) {
    const int rows = (int)src->rows, cols = (int)src->cols;
    Scratch sat;
    int rc = sat.alloc((size_t)rows * cols * CH * sizeof(float), s);
    if (rc) return rc;
    if ((rc = build_sat<PixT, CH>(src, sat.as<float>(), s))) return rc;
    const dim3 grid = row_grid(div_up((size_t)cols * CH, 256), (size_t)rows);
    sat_eval<PixT, CH, MODE><<<grid, 256, 0, s>>>(sat.as<float>(), (const PixT*)src->data, (size_t)src->stride * CH,
                                                  (PixT*)dst->data, (size_t)dst->stride * CH, rows, cols, radius, c);
    ZB_LAUNCHED();
    return ZB_OK;
}

template <int MODE>
int dispatch(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, float c, cudaStream_t s) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;  // image.zig:636,786,862
    if (MODE == EVAL_THRESHOLD && radius == 0) return ZB_ERR_INVALID_RADIUS;                 // binary.zig:93
    if (radius == 0) return zb_copy(src, dst, pixfmt, (zb_stream)s);                          // image.zig:639,789
    if ((size_t)src->rows * src->cols == 0) return ZB_OK;                                     // integral.zig:100, binary.zig:94
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if ((pixfmt == ZB_PIX_U8 || pixfmt == ZB_PIX_RGBA8) && !g_force_generic.load()) {
        rc = box_fused_u8(src, dst, pixfmt == ZB_PIX_U8 ? 1 : 4, radius, MODE + 1, c, s);
        if (rc != ZB_ERR_UNSUPPORTED) return rc;
    }
    const int rad = (int)(radius > 0x3fffffffu ? 0x3fffffffu : radius);
    if constexpr (MODE == EVAL_THRESHOLD) {
        t_last_kernel = "sat_threshold";
        return box_or_sharpen<uint8_t, 1, MODE>(src, dst, rad, c, s);
    } else {
        t_last_kernel = MODE == EVAL_SHARPEN ? "sat_sharpen" : "sat_box_blur";
        switch (pixfmt) {
            case ZB_PIX_U8: return box_or_sharpen<uint8_t, 1, MODE>(src, dst, rad, c, s);
            case ZB_PIX_F32: return box_or_sharpen<float, 1, MODE>(src, dst, rad, c, s);
            case ZB_PIX_RGB8: return box_or_sharpen<uint8_t, 3, MODE>(src, dst, rad, c, s);
            case ZB_PIX_RGBA8: return box_or_sharpen<uint8_t, 4, MODE>(src, dst, rad, c, s);
            case ZB_PIX_RGBAF32: return box_or_sharpen<float, 4, MODE>(src, dst, rad, c, s);
        }
    }
    return ZB_ERR_UNSUPPORTED;
}

}  // namespace

int sat_gray_mask(const float* gray, const uint8_t* mask, float* sat3, int rows, int cols, cudaStream_t s) {
    sat_row_pass_gray_mask<<<dim3(div_up(rows, 32), 3), 32, 0, s>>>(gray, mask, sat3, rows, cols);
    ZB_LAUNCHED();
    sat_col_pass<<<div_up((size_t)cols * 3, 256), 256, 0, s>>>(sat3, rows, cols, 3);
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace zb

using namespace zb;

extern "C" {

int zb_box_blur(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, zb_stream s) {
    return dispatch<EVAL_BOX>(src, dst, pixfmt, radius, 0.0f, (cudaStream_t)s);
}
int zb_sharpen(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius, zb_stream s) {
    return dispatch<EVAL_SHARPEN>(src, dst, pixfmt, radius, 0.0f, (cudaStream_t)s);
}
/* Image(u8).thresholdAdaptiveMean, binary.zig:86-119: the SAT and window of boxBlur (fused kernels for radius <= 15 and
 * non-overlapping buffers, the HBM summed-area table otherwise). */
int zb_threshold_adaptive_mean(const zb_image* src, zb_image* dst, uint32_t radius, float c, zb_stream s) {
    return dispatch<EVAL_THRESHOLD>(src, dst, ZB_PIX_U8, radius, c, (cudaStream_t)s);
}
int zb_integral_plane(const zb_image* src, int pixfmt, float* sat, zb_stream s) {
    if (!src || !sat) return ZB_ERR_INVALID_ARGUMENT;
    if ((size_t)src->rows * src->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (pixfmt == ZB_PIX_U8) return build_sat<uint8_t, 1>(src, sat, (cudaStream_t)s);
    if (pixfmt == ZB_PIX_F32) return build_sat<float, 1>(src, sat, (cudaStream_t)s);
    return ZB_ERR_UNSUPPORTED;
}

int zb_host_box_blur(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;
    HostStage st;
    int rc;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = zb_box_blur(&st.dsrc, &st.ddst, pixfmt, radius, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}
int zb_host_sharpen(const zb_image* src, zb_image* dst, int pixfmt, uint32_t radius) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;
    HostStage st;
    int rc;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = zb_sharpen(&st.dsrc, &st.ddst, pixfmt, radius, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

}  // extern "C"
