// zb_linalg.cu -- Matrix.gemm on the device and the Golub-Reinsch SVD on the host.
//
// GEMM (reference Matrix.zig:696-822): C = alpha * op(A) * op(B) + beta * C, all four transpose
// combinations, row-major.  The reference is a dot-product loop with f32 (or f64) accumulators whose
// summation order depends on the host's SIMD width (Matrix.zig:653-683), so it is only reproducible
// to rounding; this kernel accumulates every dot product in f64 (so an f32 GEMM is accurate to ~1e-7
// relative even for the K ~ 1e6 contractions of PCA's X^T X), tiles 64x64x16 through shared memory,
// and splits K across CTAs deterministically (partials reduced in a fixed order -- no atomics).
//
// SVD (reference svd.zig:80-496, dlib svd4 lineage): Householder bidiagonalisation + implicit-shift
// QR, descending sort.  Inherently sequential and tiny on this path (3x3 for fdm, dim x dim for pca),
// so it runs on the host; the arithmetic order is the algorithm's, which is what fixes the signs of
// the singular vectors that fdm's colour transform depends on.
#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

#include "zb_internal.h"
#include "zb_linalg.h"

namespace zb {

namespace {

constexpr int BM = 64, BN = 64, BK = 16;

template <typename T>
__global__ void __launch_bounds__(256) gemm_kernel(const T* __restrict__ A, int lda, bool ta, const T* __restrict__ B, int ldb, bool tb,
                                                   int M, int N, int K, int k_per_split, double* __restrict__ partial /* [split][M][N] */,
                                                   unsigned slices) {
    __shared__ T As[BK][BM + 1];
    __shared__ T Bs[BK][BN + 1];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = ZB_LAYER_TILE(slices) * BM, n0 = blockIdx.x * BN;
    if (m0 >= M) return;   // past the last row tile (uniform per block)
    const int split = (int)ZB_LAYER(slices);   // layered_row_grid: the K split is the layer
    const int kbeg = split * k_per_split;
    const int kend = min(K, kbeg + k_per_split);
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;

    for (int k0 = kbeg; k0 < kend; k0 += BK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + 256 * i;
            // op(A)[m][k]: contiguous along m when transposed, along k otherwise
            int m, k;
            if (ta) { m = idx & (BM - 1); k = idx >> 6; } else { k = idx & (BK - 1); m = idx >> 4; }
            const int gm = m0 + m, gk = k0 + k;
            T v = 0;
            if (gm < M && gk < kend) v = ta ? A[(size_t)gk * lda + gm] : A[(size_t)gm * lda + gk];
            As[k][m] = v;
            int n, kk;
            if (!tb) { n = idx & (BN - 1); kk = idx >> 6; } else { kk = idx & (BK - 1); n = idx >> 4; }
            const int gn = n0 + n, gkb = k0 + kk;
            T w = 0;
            if (gn < N && gkb < kend) w = tb ? B[(size_t)gn * ldb + gkb] : B[(size_t)gkb * ldb + gn];
            Bs[kk][n] = w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = (double)As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = (double)Bs[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    double* out = partial + (size_t)split * M * N;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int gm = m0 + ty * 4 + i, gn = n0 + tx * 4 + j;
            if (gm < M && gn < N) out[(size_t)gm * N + gn] = acc[i][j];
        }
}

// out = beta*c + alpha*sum_splits(partial)   (Matrix.zig:728-738, :681)
template <typename T>
__global__ void __launch_bounds__(256) gemm_finish(const double* __restrict__ partial, int splits, size_t mn, T alpha, T beta,
                                                   const T* __restrict__ c, T* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= mn) return;
    double s = 0.0;
    for (int z = 0; z < splits; ++z) s += partial[(size_t)z * mn + i];
    const T prod = (T)((double)alpha * s);
    out[i] = (c != nullptr && beta != (T)0) ? (T)(beta * c[i] + prod) : prod;
}

template <typename T>
int gemm_device(const T* a, uint32_t ar, uint32_t ac, int ta, const T* b, uint32_t br, uint32_t bc, int tb, T alpha, T beta, const T* c,
                T* out, cudaStream_t s) {
    const uint32_t a_rows = ta ? ac : ar, a_cols = ta ? ar : ac;
    const uint32_t b_rows = tb ? bc : br, b_cols = tb ? br : bc;
    if (a_cols != b_rows) return ZB_ERR_DIMENSION_MISMATCH;  // Matrix.zig:717
    if (!a || !b || !out) return ZB_ERR_INVALID_ARGUMENT;
    const int M = (int)a_rows, N = (int)b_cols, K = (int)a_cols;
    if (M == 0 || N == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if constexpr (sizeof(T) == 4) {
        // Pca.fit's covariance step (pca.zig:338): X^T X with the same matrix on both sides -> tensor cores.  The same pointer is not
        // enough: two views of one buffer may have different shapes, and the tensor-core kernel would write an ac x ac result.
        // alpha == 0 skips the product below (Matrix.zig:741); the tensor-core kernel would form it, NaN and all.
        if (ta && !tb && (const void*)a == (const void*)b && br == ar && bc == ac && alpha != (T)0 && !g_force_generic.load()) {
            rc = gemm_xtx_tensorcore((const float*)a, ar, ac, (float)alpha, (float)beta, (const float*)c, (float*)out, s);
            if (rc != ZB_ERR_UNSUPPORTED) return rc;
        }
    }
    const int tiles = div_up(M, BM) * div_up(N, BN);
    int splits = 1;
    if (K > 4 * BK) {
        splits = (2 * di.sm_count + tiles - 1) / tiles;
        const int max_splits = std::max(1, K / (8 * BK));
        splits = std::max(1, std::min(splits, max_splits));
    }
    int k_per_split = (K + splits - 1) / splits;
    k_per_split = ((k_per_split + BK - 1) / BK) * BK;
    splits = K == 0 ? 1 : (K + k_per_split - 1) / k_per_split;
    Scratch part;
    if ((rc = part.alloc((size_t)splits * M * N * sizeof(double), s))) return rc;
    if (alpha == (T)0 || K == 0) {  // Matrix.zig:741: product skipped
        ZB_CUDA(cudaMemsetAsync(part.p, 0, (size_t)splits * M * N * sizeof(double), s));
    } else {
        dim3 grid;
        unsigned slices;
        if ((rc = layered_row_grid(div_up(N, BN), div_up(M, BM), splits, &grid, &slices))) return rc;
        gemm_kernel<T><<<grid, 256, 0, s>>>(a, (int)ac, ta != 0, b, (int)bc, tb != 0, M, N, K, k_per_split, part.as<double>(), slices);
        ZB_LAUNCHED();
    }
    const size_t mn = (size_t)M * N;
    gemm_finish<T><<<div_up(mn, 256), 256, 0, s>>>(part.as<double>(), splits, mn, alpha, beta, c, out);
    ZB_LAUNCHED();
    t_last_kernel = sizeof(T) == 4 ? "gemm_f32_acc64" : "gemm_f64";
    return ZB_OK;
}


// ---- PCA centering (pca.zig:135-154): column means (f64 accumulation, deterministic two-stage) and X - mean ----
template <typename T>
__global__ void __launch_bounds__(256) colsum_kernel(const T* __restrict__ x, uint32_t n, uint32_t dim, uint32_t rows_per_block,
                                                     double* __restrict__ partial /* [gridDim.y][dim] */) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= dim) return;
    const uint32_t r0 = blockIdx.y * rows_per_block;
    const uint32_t r1 = min(n, r0 + rows_per_block);
    double s = 0.0;
    for (uint32_t i = r0; i < r1; ++i) s += (double)x[(size_t)i * dim + j];
    partial[(size_t)blockIdx.y * dim + j] = s;
}
template <typename T>
__global__ void __launch_bounds__(256) colmean_finish(const double* __restrict__ partial, uint32_t parts, uint32_t n, uint32_t dim,
                                                      T* __restrict__ mean) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= dim) return;
    double s = 0.0;
    for (uint32_t p = 0; p < parts; ++p) s += partial[(size_t)p * dim + j];
    mean[j] = (T)(s / (double)n);
}
template <typename T>
__global__ void __launch_bounds__(256) center_kernel(const T* __restrict__ x, const T* __restrict__ mean, size_t total, uint32_t dim,
                                                     T* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    out[i] = x[i] - mean[i % dim];
}

template <typename T>
int center_columns(const T* x, uint32_t n, uint32_t dim, T* mean, int compute_mean, T* centered, cudaStream_t s) {
    if (!x || !mean) return ZB_ERR_INVALID_ARGUMENT;
    if (n == 0 || dim == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (compute_mean) {
        const uint32_t col_blocks = div_up(dim, 256);
        uint32_t parts = std::max<uint32_t>(1, (uint32_t)(4 * di.sm_count) / col_blocks);
        parts = std::min<uint32_t>(parts, std::max<uint32_t>(1, n / 64));
        const uint32_t rows_per_block = (n + parts - 1) / parts;
        parts = (n + rows_per_block - 1) / rows_per_block;
        Scratch part;
        if ((rc = part.alloc((size_t)parts * dim * sizeof(double), s))) return rc;
        colsum_kernel<T><<<dim3(col_blocks, parts), 256, 0, s>>>(x, n, dim, rows_per_block, part.as<double>());
        ZB_LAUNCHED();
        colmean_finish<T><<<col_blocks, 256, 0, s>>>(part.as<double>(), parts, n, dim, mean);
        ZB_LAUNCHED();
    }
    if (centered) {
        const size_t total = (size_t)n * dim;
        center_kernel<T><<<div_up(total, 256), 256, 0, s>>>(x, mean, total, dim, centered);
        ZB_LAUNCHED();
    }
    return ZB_OK;
}

}  // namespace

}  // namespace zb

using namespace zb;

extern "C" {

int zb_gemm_f32(const float* a, uint32_t ar, uint32_t ac, int ta, const float* b, uint32_t br, uint32_t bc, int tb, float alpha, float beta,
                const float* c, float* out, zb_stream s) {
    return gemm_device<float>(a, ar, ac, ta, b, br, bc, tb, alpha, beta, c, out, (cudaStream_t)s);
}
int zb_gemm_f64(const double* a, uint32_t ar, uint32_t ac, int ta, const double* b, uint32_t br, uint32_t bc, int tb, double alpha,
                double beta, const double* c, double* out, zb_stream s) {
    return gemm_device<double>(a, ar, ac, ta, b, br, bc, tb, alpha, beta, c, out, (cudaStream_t)s);
}
int zb_center_columns_f32(const float* x, uint32_t n, uint32_t dim, float* mean, int compute_mean, float* centered, zb_stream s) {
    return center_columns<float>(x, n, dim, mean, compute_mean, centered, (cudaStream_t)s);
}
int zb_center_columns_f64(const double* x, uint32_t n, uint32_t dim, double* mean, int compute_mean, double* centered, zb_stream s) {
    return center_columns<double>(x, n, dim, mean, compute_mean, centered, (cudaStream_t)s);
}

}  // extern "C"
