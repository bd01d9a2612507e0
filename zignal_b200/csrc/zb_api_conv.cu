// zb_api_conv.cu -- C entry points for Image.convolveSeparable / convolve / gaussianBlur
// (reference image.zig:917-994, convolution.zig:198-438) and their host-pointer twins.
#include <algorithm>
#include <cmath>
#include <vector>

#include "zb_conv.h"
#include "zb_host_stage.h"

using namespace zb;

namespace zb {

static int check_shapes(const zb_image* src, const zb_image* dst, int pixfmt) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmtAll, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;  // image.zig:927,947,962
    return ZB_OK;
}

// Output rows [row0, row1) only (row1 < 0: all rows).
int conv_separable_dispatch(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny,
                            int border, cudaStream_t s, int row0 = 0, int row1 = -1) {
    int rc = check_shapes(src, dst, pixfmt);
    if (rc) return rc;
    if (exceeds_int_index(src, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (nx <= 0 || ny <= 0 || !kx || !ky) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    if (row1 < 0 || row1 > (int)src->rows) row1 = (int)src->rows;
    if (row0 < 0 || row0 > row1) return ZB_ERR_INVALID_ARGUMENT;
    if (row0 == row1) return ZB_OK;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;
    if (pixfmt == ZB_PIX_RGBAF32 && !g_force_generic.load()) {
        rc = conv_separable_fused_rgbaf32(src, dst, kx, nx, ky, ny, border, g_exact_f32.load() != 0, s, row0, row1);
        if (rc != ZB_ERR_UNSUPPORTED) return rc;
    }
    if (pixfmt == ZB_PIX_RGBA8 && !g_force_generic.load()) {
        rc = conv_separable_fused_rgba8(src, dst, kx, nx, ky, ny, border, s, row0, row1);
        if (rc != ZB_ERR_UNSUPPORTED) return rc;
    }
    if (row0 == 0 && row1 == (int)src->rows) {
        if (pixfmt_in(kFmt8Bit, pixfmt) && !g_force_generic.load()) {
            rc = conv_separable_tile_u8(src, dst, channels_of(pixfmt), kx, nx, ky, ny, border, s);
            if (rc != ZB_ERR_UNSUPPORTED) return rc;
        }
        return conv_separable_generic(src, dst, pixfmt, kx, nx, ky, ny, border, s);
    }
    // two-pass path: it has no row window, so convolve into scratch and keep the requested rows
    const size_t pb = pixel_bytes(pixfmt);
    Scratch tmp;
    if ((rc = tmp.alloc((size_t)src->rows * src->cols * pb, s))) return rc;
    zb_image full{tmp.p, src->rows, src->cols, src->cols};
    if ((rc = conv_separable_generic(src, &full, pixfmt, kx, nx, ky, ny, border, s))) return rc;
    if ((rc = span_copy((char*)dst->data + (size_t)row0 * dst->stride * pb, dst->stride * pb, (char*)tmp.p + (size_t)row0 * src->cols * pb,
                        (size_t)src->cols * pb, (size_t)src->cols * pb, (size_t)(row1 - row0), cudaMemcpyDeviceToDevice, s))) return rc;
    return ZB_OK;
}

// image.zig:972-990
int gaussian_taps_host(float sigma, std::vector<float>& taps) {
    // image.zig:973 casts ceil(3 sigma) to usize: a NaN / infinite sigma is a panic there, an error code here; a radius beyond 2^24
    // could not be allocated either (and no kernel of this build takes it)
    if (!std::isfinite(sigma)) return ZB_ERR_INVALID_SIGMA;
    if (3.0f * sigma > 16777216.0f) return ZB_ERR_UNSUPPORTED;
    const size_t radius = (size_t)std::ceil(3.0f * sigma);
    const size_t n = 2 * radius + 1;
    taps.resize(n);
    float sum = 0;
    for (size_t i = 0; i < n; ++i) {
        const float x = (float)i - (float)radius;
        taps[i] = std::exp(-(x * x) / (2.0f * sigma * sigma));
        sum += taps[i];
    }
    for (size_t i = 0; i < n; ++i) taps[i] /= sum;
    return ZB_OK;
}

}  // namespace zb

// ---------------------------------------------------------------------------------------------------------------
// Pipelined host path for the fused single-pass kernels: the image crosses PCIe in row bands on one stream, each
// band is convolved on a second stream as soon as the rows it reads (itself plus `half` rows of the next band) have
// landed, and finished bands go back on a third stream -- PCIe is full duplex, so the call costs about one
// direction's transfer time instead of H2D + kernel + D2H back to back.  Results are identical to the one-shot
// path: every launch sees the whole source image, only its OUTPUT rows are restricted.
// ---------------------------------------------------------------------------------------------------------------
namespace {

struct PipeStreams {
    cudaStream_t up = nullptr, run = nullptr, down = nullptr;
    int device = -1;
};
thread_local PipeStreams t_pipe;

int pipe_streams(PipeStreams** out) {
    int dev = 0;
    ZB_CUDA(cudaGetDevice(&dev));
    if (t_pipe.device != dev) {
        // (streams of a previous device, if any, are leaked on purpose: destroying them needs that device current)
        ZB_CUDA(cudaStreamCreateWithFlags(&t_pipe.up, cudaStreamNonBlocking));
        ZB_CUDA(cudaStreamCreateWithFlags(&t_pipe.run, cudaStreamNonBlocking));
        ZB_CUDA(cudaStreamCreateWithFlags(&t_pipe.down, cudaStreamNonBlocking));
        t_pipe.device = dev;
    }
    *out = &t_pipe;
    return ZB_OK;
}

struct EventList {
    std::vector<cudaEvent_t> ev;
    ~EventList() { for (cudaEvent_t e : ev) cudaEventDestroy(e); }
    int make(cudaEvent_t* e) {
        ZB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
        ev.push_back(*e);
        return ZB_OK;
    }
};

}  // namespace

// Returns ZB_ERR_UNSUPPORTED when the configuration has no fused kernel (the caller then stages the whole image).
static int host_conv_separable_pipelined(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny,
                                         int border) {
    if (pixfmt != ZB_PIX_RGBAF32 && pixfmt != ZB_PIX_RGBA8) return ZB_ERR_UNSUPPORTED;
    if (g_force_generic.load() || border == ZB_BORDER_WRAP) return ZB_ERR_UNSUPPORTED;   // wrap: the first band reads the last rows
    if (nx <= 0 || ny <= 0 || !kx || !ky) return ZB_ERR_INVALID_ARGUMENT;
    const size_t pb = pixel_bytes(pixfmt);
    const int rows = (int)src->rows, cols = (int)src->cols;
    const int half = ny / 2;
    int band = g_tune_host_band_rows.load();
    if (band <= 0) return ZB_ERR_UNSUPPORTED;
    band = (band + 63) / 64 * 64;
    if (rows < 2 * band || half >= band || (size_t)rows * cols * pb < ((size_t)32 << 20)) return ZB_ERR_UNSUPPORTED;  // small: one shot
    PipeStreams* ps;
    int rc = pipe_streams(&ps);
    if (rc) return rc;
    Scratch s_src, s_dst;
    if ((rc = s_src.alloc((size_t)rows * cols * pb, ps->up))) return rc;
    if ((rc = s_dst.alloc((size_t)rows * cols * pb, ps->up))) return rc;
    const zb_image dsrc{s_src.p, src->rows, src->cols, src->cols};
    zb_image ddst{s_dst.p, dst->rows, dst->cols, dst->cols};
    EventList evs;
    cudaEvent_t e_alloc;
    if ((rc = evs.make(&e_alloc))) return rc;
    ZB_CUDA(cudaEventRecord(e_alloc, ps->up));
    ZB_CUDA(cudaStreamWaitEvent(ps->run, e_alloc, 0));
    const int nb = (rows + band - 1) / band;
    const bool exact = g_exact_f32.load() != 0;
    auto run_band = [&](int j, cudaEvent_t uploaded) -> int {
        const int y0 = j * band, y1 = std::min(rows, y0 + band);
        ZB_CUDA(cudaStreamWaitEvent(ps->run, uploaded, 0));
        int r = pixfmt == ZB_PIX_RGBAF32 ? conv_separable_fused_rgbaf32(&dsrc, &ddst, kx, nx, ky, ny, border, exact, ps->run, y0, y1)
                                         : conv_separable_fused_rgba8(&dsrc, &ddst, kx, nx, ky, ny, border, ps->run, y0, y1);
        if (r) return r;
        cudaEvent_t done;
        if ((r = evs.make(&done))) return r;
        ZB_CUDA(cudaEventRecord(done, ps->run));
        ZB_CUDA(cudaStreamWaitEvent(ps->down, done, 0));
        return span_copy((char*)dst->data + (size_t)y0 * dst->stride * pb, dst->stride * pb, (char*)s_dst.p + (size_t)y0 * cols * pb,
                         (size_t)cols * pb, (size_t)cols * pb, (size_t)(y1 - y0), cudaMemcpyDeviceToHost, ps->down);
    };
    cudaEvent_t prev_up = nullptr;
    for (int j = 0; j < nb; ++j) {
        const int y0 = j * band, y1 = std::min(rows, y0 + band);
        if ((rc = span_copy((char*)s_src.p + (size_t)y0 * cols * pb, (size_t)cols * pb, (const char*)src->data + (size_t)y0 * src->stride * pb,
                            src->stride * pb, (size_t)cols * pb, (size_t)(y1 - y0), cudaMemcpyHostToDevice, ps->up))) return rc;
        cudaEvent_t up;
        if ((rc = evs.make(&up))) return rc;
        ZB_CUDA(cudaEventRecord(up, ps->up));
        if (j > 0) {
            rc = run_band(j - 1, up);   // band j-1 reads up to `half` rows of band j
            if (rc == ZB_ERR_UNSUPPORTED && j == 1) {   // outside the fused envelope: nothing has been computed yet
                ZB_CUDA(cudaStreamSynchronize(ps->up));
                return rc;
            }
            if (rc) { cudaDeviceSynchronize(); return rc; }
        }
        prev_up = up;
    }
    if ((rc = run_band(nb - 1, prev_up))) { cudaDeviceSynchronize(); return rc; }
    ZB_CUDA(cudaStreamSynchronize(ps->down));
    ZB_CUDA(cudaStreamSynchronize(ps->run));
    return ZB_OK;
}

extern "C" {

int zb_gaussian_taps(float sigma, float* taps, int cap, int* n) {
    if (!n) return ZB_ERR_INVALID_ARGUMENT;
    if (sigma == 0) { *n = 0; return ZB_OK; }
    if (!(sigma > 0)) return ZB_ERR_INVALID_SIGMA;
    std::vector<float> t;
    if (int rc = gaussian_taps_host(sigma, t)) return rc;
    *n = (int)t.size();
    if (!taps || cap < (int)t.size()) return ZB_ERR_INVALID_ARGUMENT;
    memcpy(taps, t.data(), t.size() * sizeof(float));
    return ZB_OK;
}

int zb_conv_separable(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny, int border,
                      zb_stream s) {
    return conv_separable_dispatch(src, dst, pixfmt, kx, nx, ky, ny, border, (cudaStream_t)s);
}

int zb_conv_separable_rows(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny, int border,
                           uint32_t row_begin, uint32_t row_end, zb_stream s) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (row_end == 0 || row_end > src->rows) row_end = src->rows;
    if (row_begin > row_end) return ZB_ERR_INVALID_ARGUMENT;
    if (images_overlap(src, dst, pixel_bytes(pixfmt))) return ZB_ERR_INVALID_ARGUMENT;   // a row window of an in-place convolution would read rows already overwritten
    return conv_separable_dispatch(src, dst, pixfmt, kx, nx, ky, ny, border, (cudaStream_t)s, (int)row_begin, (int)row_end);
}

int zb_convolve(const zb_image* src, zb_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border, zb_stream s) {
    int rc = check_shapes(src, dst, pixfmt);
    if (rc) return rc;
    if (exceeds_int_index(src, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (kh <= 0 || kw <= 0 || !kernel) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;
    return convolve_generic(src, dst, pixfmt, kernel, kh, kw, border, (cudaStream_t)s);
}

int zb_gaussian_blur(const zb_image* src, zb_image* dst, int pixfmt, float sigma, zb_stream s) {
    int rc = check_shapes(src, dst, pixfmt);
    if (rc) return rc;
    if (sigma == 0) return zb_copy(src, dst, pixfmt, s);   // image.zig:966
    if (exceeds_int_index(src, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (!(sigma > 0)) return ZB_ERR_INVALID_SIGMA;         // image.zig:970
    std::vector<float> taps;
    if ((rc = gaussian_taps_host(sigma, taps))) return rc;
    return conv_separable_dispatch(src, dst, pixfmt, taps.data(), (int)taps.size(), taps.data(), (int)taps.size(), ZB_BORDER_MIRROR,
                                   (cudaStream_t)s);     // image.zig:993
}

int zb_host_conv_separable(const zb_image* src, zb_image* dst, int pixfmt, const float* kx, int nx, const float* ky, int ny,
                           int border) {
    int rc = check_shapes(src, dst, pixfmt);
    if (rc) return rc;
    if (exceeds_int_index(src, pixfmt)) return ZB_ERR_UNSUPPORTED;   // before staging
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    rc = host_conv_separable_pipelined(src, dst, pixfmt, kx, nx, ky, ny, border);
    if (rc != ZB_ERR_UNSUPPORTED) return rc;
    HostStage st;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = conv_separable_dispatch(&st.dsrc, &st.ddst, pixfmt, kx, nx, ky, ny, border, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

int zb_host_convolve(const zb_image* src, zb_image* dst, int pixfmt, const float* kernel, int kh, int kw, int border) {
    int rc = check_shapes(src, dst, pixfmt);
    if (rc) return rc;
    if (exceeds_int_index(src, pixfmt)) return ZB_ERR_UNSUPPORTED;   // before staging
    HostStage st;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = zb_convolve(&st.dsrc, &st.ddst, pixfmt, kernel, kh, kw, border, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

int zb_host_gaussian_blur(const zb_image* src, zb_image* dst, int pixfmt, float sigma) {
    int rc = check_shapes(src, dst, pixfmt);
    if (rc) return rc;
    if (exceeds_int_index(src, pixfmt)) return ZB_ERR_UNSUPPORTED;   // before staging
    if (!(sigma >= 0)) return ZB_ERR_INVALID_SIGMA;
    if (sigma > 0) {
        std::vector<float> taps;
        if ((rc = gaussian_taps_host(sigma, taps))) return rc;
        rc = host_conv_separable_pipelined(src, dst, pixfmt, taps.data(), (int)taps.size(), taps.data(), (int)taps.size(), ZB_BORDER_MIRROR);
        if (rc != ZB_ERR_UNSUPPORTED) return rc;
    }
    HostStage st;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = zb_gaussian_blur(&st.dsrc, &st.ddst, pixfmt, sigma, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

}  // extern "C"
