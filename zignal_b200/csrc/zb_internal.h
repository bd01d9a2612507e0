// zb_internal.h -- shared internals of libzignal_b200.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../../include/zignal_b200.h"

namespace zb {

extern std::atomic<uint64_t> g_launches;
extern thread_local char t_last_error[512];
extern thread_local const char* t_last_kernel;
extern std::atomic<int> g_exact_f32;
extern std::atomic<int> g_force_generic;
extern std::atomic<int> g_tune_band_rows;  // sharded fused RGBA f32 conv: target rows per band (the single-GPU kernels plan their own rows)
extern std::atomic<int> g_tune_host_band_rows;  // host-pointer pipeline: rows per PCIe band (0 disables the pipeline)
extern std::atomic<int> g_tune_edge_fast;  // fused RGBA f32 conv: x borders of .replicate / .mirror as in-stage copies (default on; 0 = generic fixup pass)
extern std::atomic<int> g_tune_sobel_tile; // Image.sobel on gray u8: byte-tile kernel (default on; 0 = per-pixel kernel)
extern std::atomic<int> g_tune_jacobi_cluster;  // Jacobi SVD in one cluster's distributed shared memory when it fits (default on)
extern std::atomic<int> g_tune_u8_dp;      // fused RGBA8 conv: dp4a / dp2a variant when every tap is a byte (default on)
extern std::atomic<int> g_tune_u8_fmath;   // fused RGBA8 conv: run the exact-integer pipeline on FFMA when provably exact

int set_cuda_error(cudaError_t e, const char* what, const char* file, int line);

#define ZB_CUDA(expr)                                                                    \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) return ::zb::set_cuda_error(_e, #expr, __FILE__, __LINE__); \
    } while (0)

// Count + check a kernel launch.
#define ZB_LAUNCHED()                                                                      \
    do {                                                                                   \
        ::zb::g_launches.fetch_add(1, std::memory_order_relaxed);                          \
        cudaError_t _e = cudaGetLastError();                                               \
        if (_e != cudaSuccess) return ::zb::set_cuda_error(_e, "kernel launch", __FILE__, __LINE__); \
    } while (0)

struct DeviceInfo {
    int ordinal = -1;
    int sm_count = 0;
    size_t smem_optin = 0;
};
// Lazily initialised per-device state (mempool threshold, SM count, driver entry points).
int device_info(DeviceInfo* out);
// cuTensorMapEncodeTiled resolved through cudaGetDriverEntryPoint (no link-time libcuda dependency).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn();

static inline int channels_of(int pixfmt) {
    switch (pixfmt) {
        case ZB_PIX_U8: case ZB_PIX_F32: return 1;
        case ZB_PIX_RGB8: return 3;
        case ZB_PIX_RGBA8: case ZB_PIX_RGBAF32: return 4;
    }
    return 0;
}
static inline size_t channel_bytes(int pixfmt) { return (pixfmt == ZB_PIX_F32 || pixfmt == ZB_PIX_RGBAF32) ? 4 : 1; }
static inline size_t pixel_bytes(int pixfmt) { return (size_t)channels_of(pixfmt) * channel_bytes(pixfmt); }
static inline bool is_float_fmt(int pixfmt) { return pixfmt == ZB_PIX_F32 || pixfmt == ZB_PIX_RGBAF32; }

// RAII stream-ordered scratch (cudaMallocAsync / cudaFreeAsync on the op's stream).
struct Scratch {
    void* p = nullptr;
    cudaStream_t s = nullptr;
    ~Scratch() { if (p) cudaFreeAsync(p, s); }
    int alloc(size_t bytes, cudaStream_t stream);
    template <typename T> T* as() const { return (T*)p; }
};

// Do the byte ranges two image views span intersect?  (Two views of one buffer with different base pointers may still
// overlap; single-pass kernels read neighbourhoods other blocks are writing, so any overlap must take the snapshot path.)
static inline bool images_overlap(const zb_image* a, const zb_image* b, size_t pixel_bytes_) {
    if (!a->data || !b->data || a->rows == 0 || a->cols == 0 || b->rows == 0 || b->cols == 0) return false;
    const uintptr_t a0 = (uintptr_t)a->data, b0 = (uintptr_t)b->data;
    const uintptr_t a1 = a0 + ((size_t)(a->rows - 1) * a->stride + a->cols) * pixel_bytes_;
    const uintptr_t b1 = b0 + ((size_t)(b->rows - 1) * b->stride + b->cols) * pixel_bytes_;
    return a0 < b1 && b0 < a1;
}

static inline unsigned div_up(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

// zb_integral.cu: the three f32 summed-area tables of Shen-Castan's adaptive gradient (edges.zig:434-452) into sat3 (3 x rows x cols,
// contiguous): plane 0 of gray, plane 1 of the 0 / 1 mask, plane 2 of gray * mask.  The row and column passes of Image.integral, so the
// order of additions is the reference's (integral.zig:41-78).  gray and mask are rows x cols contiguous device planes.
int sat_gray_mask(const float* gray, const uint8_t* mask, float* sat3, int rows, int cols, cudaStream_t s);

// The one mapping of row tiles onto the grid.  gridDim.y is capped at 65,535, so a launch with one block row per image row (or
// per tile of rows) spreads the tiles over (y, z): row_grid(x_blocks, n_tiles) and ZB_GRID_ROW() as the tile index.  Kernels
// return at their top when the tile index is >= the tile count (the last z-slice may be partly empty); that test is uniform per
// block, so it may precede __syncthreads.
//
// Kernels that already use z for a layer (the frame of a batch, the K split of a GEMM) take layered_row_grid: z = layer * slices
// + slice, the tile index is ZB_LAYER_TILE(slices) and the layer ZB_LAYER(slices).  It refuses (ZB_ERR_UNSUPPORTED) when
// layers * slices would exceed gridDim.z's 65,535, i.e. beyond 65,535 x 65,535 tiles in all.
#ifdef __CUDACC__
#define ZB_GRID_ROW() ((int)(blockIdx.y + blockIdx.z * gridDim.y))
#define ZB_LAYER_TILE(slices) ((int)(blockIdx.y + (blockIdx.z % (slices)) * gridDim.y))
#define ZB_LAYER(slices) (blockIdx.z / (slices))
static inline dim3 row_grid(unsigned x_blocks, size_t rows) {
    const size_t gz = (rows + 65534) / 65535;
    const size_t gy = gz ? (rows + gz - 1) / gz : 0;
    return dim3(x_blocks, (unsigned)gy, (unsigned)(gz ? gz : 1));
}
static inline int layered_row_grid(unsigned x_blocks, size_t n_tiles, size_t layers, dim3* grid, unsigned* slices) {
    const dim3 g = row_grid(x_blocks, n_tiles);
    if ((size_t)g.z * layers > 65535u) return ZB_ERR_UNSUPPORTED;
    *grid = dim3(g.x, g.y, (unsigned)(g.z * layers));
    *slices = g.z;
    return ZB_OK;
}
#endif

}  // namespace zb
