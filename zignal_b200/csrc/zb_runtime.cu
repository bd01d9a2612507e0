// zb_runtime.cu -- device / stream / memory plumbing behind the C ABI (include/zignal_b200.h).
// These wrappers are what the Zig shim's DeviceAllocator (std.mem.Allocator vtable) and
// Image(T).init/deinit (reference image.zig:124-158) sit on.
#include <mutex>

#include "zb_internal.h"

namespace zb {

std::atomic<uint64_t> g_launches{0};
thread_local char t_last_error[512] = "";
thread_local const char* t_last_kernel = "";
std::atomic<int> g_exact_f32{0};
std::atomic<int> g_force_generic{0};
std::atomic<int> g_tune_band_rows{256};
std::atomic<int> g_tune_host_band_rows{256};
std::atomic<int> g_tune_u8_fmath{1};
std::atomic<int> g_tune_u8_dp{1};
std::atomic<int> g_tune_rotate_tile{1};
std::atomic<int> g_tune_edge_fast{1};
std::atomic<int> g_tune_sobel_tile{1};
std::atomic<int> g_tune_jacobi_cluster{1};

int set_cuda_error(cudaError_t e, const char* what, const char* file, int line) {
    snprintf(t_last_error, sizeof(t_last_error), "%s: %s (%s:%d)", cudaGetErrorName(e), what, file, line);
    if (e == cudaErrorMemoryAllocation) return ZB_ERR_OUT_OF_MEMORY;
    return ZB_ERR_DEVICE_FAILURE;
}

static std::mutex g_mu;
static DeviceInfo g_dev[64];
static EncodeTiledFn g_encode = nullptr;

int device_info(DeviceInfo* out) {
    int dev = 0;
    ZB_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) return ZB_ERR_DEVICE_FAILURE;
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_dev[dev].ordinal != dev) {
        cudaDeviceProp prop;
        ZB_CUDA(cudaGetDeviceProperties(&prop, dev));
        g_dev[dev].sm_count = prop.multiProcessorCount;
        g_dev[dev].smem_optin = prop.sharedMemPerBlockOptin;
        // keep freed scratch cached in the default pool instead of returning it to the driver
        cudaMemPool_t pool;
        ZB_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
        uint64_t thresh = UINT64_MAX;
        ZB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
        g_dev[dev].ordinal = dev;
    }
    *out = g_dev[dev];
    return ZB_OK;
}

EncodeTiledFn encode_tiled_fn() {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            g_encode = (EncodeTiledFn)fn;
    }
    return g_encode;
}

int Scratch::alloc(size_t bytes, cudaStream_t stream) {
    s = stream;
    if (bytes == 0) bytes = 16;
    ZB_CUDA(cudaMallocAsync(&p, bytes, stream));
    return ZB_OK;
}

}  // namespace zb

using namespace zb;

extern "C" {

int zb_version(void) { return ZB_VERSION_MAJOR * 1000 + ZB_VERSION_MINOR; }

const char* zb_status_name(int status) {
    switch (status) {
        case ZB_OK: return "Ok";
        case ZB_ERR_DIMENSION_MISMATCH: return "DimensionMismatch";
        case ZB_ERR_INVALID_SIGMA: return "InvalidSigma";
        case ZB_ERR_UNSUPPORTED: return "Unsupported";
        case ZB_ERR_NOT_CONVERGED: return "NotConverged";
        case ZB_ERR_INVALID_ARGUMENT: return "InvalidArgument";
        case ZB_ERR_OUT_OF_MEMORY: return "OutOfMemory";
        case ZB_ERR_DEVICE_FAILURE: return "DeviceFailure";
        case ZB_ERR_INVALID_SCALE_FACTOR: return "InvalidScaleFactor";
        case ZB_ERR_INVALID_DIMENSIONS: return "InvalidDimensions";
        case ZB_ERR_NO_TARGET_SET: return "NoTargetSet";
        case ZB_ERR_NO_SOURCE_SET: return "NoSourceSet";
        case ZB_ERR_INSUFFICIENT_DATA: return "InsufficientData";
        case ZB_ERR_INVALID_COMPONENTS: return "InvalidComponents";
        case ZB_ERR_INVALID_THRESHOLD: return "InvalidThreshold";
        case ZB_ERR_INVALID_PERCENTILE: return "InvalidPercentile";
        case ZB_ERR_INVALID_TRIM: return "InvalidTrim";
        case ZB_ERR_IMAGE_TOO_SMALL: return "ImageTooSmall";
        case ZB_ERR_NOT_SQUARE: return "NotSquare";
        case ZB_ERR_NOT_SYMMETRIC: return "NotSymmetric";
        case ZB_ERR_NOT_FINITE: return "NotFinite";
        case ZB_ERR_INVALID_CUTOFF: return "InvalidCutoff";
        case ZB_ERR_INVALID_RADIUS: return "InvalidRadius";
        case ZB_ERR_INVALID_KERNEL_SIZE: return "InvalidKernelSize";
        case ZB_ERR_INVALID_B_PARAMETER: return "InvalidBParameter";
        case ZB_ERR_WINDOW_SIZE_MUST_BE_ODD: return "WindowSizeMustBeOdd";
        case ZB_ERR_WINDOW_SIZE_TOO_SMALL: return "WindowSizeTooSmall";
    }
    return "Unknown";
}

const char* zb_last_error(void) { return t_last_error; }
const char* zb_last_kernel(void) { return t_last_kernel; }
uint64_t zb_kernel_launch_count(void) { return g_launches.load(); }
int zb_set_exact_f32(int on) { g_exact_f32.store(on ? 1 : 0); return ZB_OK; }
int zb_set_force_generic(int on) { g_force_generic.store(on ? 1 : 0); return ZB_OK; }
int zb_tune(const char* key, int value) {
    if (!key) return ZB_ERR_INVALID_ARGUMENT;
    if (!strcmp(key, "conv.u8_fmath")) { g_tune_u8_fmath.store(value ? 1 : 0); return ZB_OK; }
    if (!strcmp(key, "conv.u8_dp")) { g_tune_u8_dp.store(value ? 1 : 0); return ZB_OK; }
    if (!strcmp(key, "conv.edge_fast")) { g_tune_edge_fast.store(value ? 1 : 0); return ZB_OK; }
    if (!strcmp(key, "sobel.tile")) { g_tune_sobel_tile.store(value ? 1 : 0); return ZB_OK; }
    if (!strcmp(key, "jacobi.cluster")) { g_tune_jacobi_cluster.store(value ? 1 : 0); return ZB_OK; }
    if (!strcmp(key, "rotate.tile")) { g_tune_rotate_tile.store(value ? 1 : 0); return ZB_OK; }
    if (!strcmp(key, "host.band_rows")) { if (value < 0) return ZB_ERR_INVALID_ARGUMENT; g_tune_host_band_rows.store(value); return ZB_OK; }
    if (!strcmp(key, "conv.band_rows")) { if (value < 64) return ZB_ERR_INVALID_ARGUMENT; g_tune_band_rows.store(value); return ZB_OK; }
    return ZB_ERR_INVALID_ARGUMENT;
}

int zb_device_count(int* count) { ZB_CUDA(cudaGetDeviceCount(count)); return ZB_OK; }
int zb_set_device(int ordinal) { ZB_CUDA(cudaSetDevice(ordinal)); return ZB_OK; }
int zb_get_device(int* ordinal) { ZB_CUDA(cudaGetDevice(ordinal)); return ZB_OK; }
int zb_sm_count(int* count) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    *count = di.sm_count;
    return ZB_OK;
}

int zb_stream_create(zb_stream* out) {
    cudaStream_t s;
    ZB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    *out = (zb_stream)s;
    return ZB_OK;
}
int zb_stream_destroy(zb_stream s) { ZB_CUDA(cudaStreamDestroy((cudaStream_t)s)); return ZB_OK; }
int zb_stream_synchronize(zb_stream s) { ZB_CUDA(cudaStreamSynchronize((cudaStream_t)s)); return ZB_OK; }

int zb_malloc(void** out, size_t bytes, zb_stream s) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (bytes == 0) bytes = 16;
    ZB_CUDA(cudaMallocAsync(out, bytes, (cudaStream_t)s));
    return ZB_OK;
}
int zb_free(void* p, zb_stream s) {
    if (!p) return ZB_OK;
    ZB_CUDA(cudaFreeAsync(p, (cudaStream_t)s));
    return ZB_OK;
}
int zb_malloc_host(void** out, size_t bytes) {
    ZB_CUDA(cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocDefault));
    return ZB_OK;
}
int zb_free_host(void* p) {
    if (!p) return ZB_OK;
    ZB_CUDA(cudaFreeHost(p));
    return ZB_OK;
}

static int copy2d(const zb_image* src, zb_image* dst, int pixfmt, cudaMemcpyKind kind, cudaStream_t s) {
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;
    const size_t pb = pixel_bytes(pixfmt);
    if (pb == 0) return ZB_ERR_UNSUPPORTED;
    if (src->rows == 0 || src->cols == 0) return ZB_OK;
    if (src->data == dst->data) return ZB_OK;  // image.zig:377
    ZB_CUDA(cudaMemcpy2DAsync(dst->data, dst->stride * pb, src->data, src->stride * pb, (size_t)src->cols * pb, src->rows, kind, s));
    return ZB_OK;
}
int zb_set_border_zero(zb_image* img, int pixfmt, uint32_t l, uint32_t t, uint32_t r, uint32_t b, zb_stream s) {
    if (!img) return ZB_ERR_INVALID_ARGUMENT;
    const size_t pb = pixel_bytes(pixfmt);
    if (pb == 0) return ZB_ERR_UNSUPPORTED;
    if (img->rows == 0 || img->cols == 0) return ZB_OK;
    r = r < img->cols ? r : img->cols;   // bounds.intersect(rect)
    b = b < img->rows ? b : img->rows;
    if (l >= r || t >= b) { l = r = 0; t = b = 0; }   // no intersection: everything is border (image.zig:202-205)
    char* base = (char*)img->data;
    const size_t pitch = img->stride * pb;
    auto zero = [&](uint32_t row0, uint32_t row1, uint32_t col0, uint32_t col1) -> int {
        if (row1 <= row0 || col1 <= col0) return ZB_OK;
        ZB_CUDA(cudaMemset2DAsync(base + (size_t)row0 * pitch + (size_t)col0 * pb, pitch, 0, (size_t)(col1 - col0) * pb, row1 - row0, (cudaStream_t)s));
        return ZB_OK;
    };
    int rc;
    if ((rc = zero(0, t, 0, img->cols))) return rc;           // top band
    if ((rc = zero(t, b, 0, l))) return rc;                   // left of the rect
    if ((rc = zero(t, b, r, img->cols))) return rc;           // right of the rect
    return zero(b, img->rows, 0, img->cols);                  // bottom band
}

int zb_upload(const zb_image* host_src, zb_image* dev_dst, int pixfmt, zb_stream s) {
    return copy2d(host_src, dev_dst, pixfmt, cudaMemcpyHostToDevice, (cudaStream_t)s);
}
int zb_download(const zb_image* dev_src, zb_image* host_dst, int pixfmt, zb_stream s) {
    return copy2d(dev_src, host_dst, pixfmt, cudaMemcpyDeviceToHost, (cudaStream_t)s);
}
int zb_copy(const zb_image* dev_src, zb_image* dev_dst, int pixfmt, zb_stream s) {
    return copy2d(dev_src, dev_dst, pixfmt, cudaMemcpyDeviceToDevice, (cudaStream_t)s);
}

}  // extern "C"
