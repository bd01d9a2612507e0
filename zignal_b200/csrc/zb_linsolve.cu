// zb_linsolve.cu -- Matrix.lu / LuResult.solve / det / inv / chol (reference Matrix.zig:67-85, 376-441, 511-583, 1156-1365) on the
// device, as blocked factorisations with panel width NB = 64:
//
//   panel      one cooperative launch per NB columns.  Each CTA holds a contiguous slab of the panel's rows in shared memory; per
//              column every CTA publishes its arg-max candidate row (and the owner of the pivot position publishes that row), one
//              grid barrier, then every CTA picks the same winner and eliminates its own rows.  The arithmetic is the reference's
//              loop body in its order (division, then subtraction without contraction; the `|pivot| > eps` rule; Gauss-Jordan's
//              scaling of the pivot row by division).  The arg-max keeps the first maximal row and maps NaN below every number, so
//              a NaN only ends up as pivot when it is on the diagonal -- the reference's sequential `>` scan.
//   swaps      the panel's interchanges, applied to every column outside it (one thread per column).
//   block row  LU: U12 = L11^-1 A12 in the reference's subtraction order; Gauss-Jordan: the NB pivot rows of every column outside the
//              panel (scale, eliminate the other block rows); Cholesky: L21 = A21 L11^-T row by row.  One thread per column (row).
//   update     C -= A B with A of width NB: f64 on the FP64 tensor cores (mma.m16n8k16 -> DMMA), f32 on FFMA with f32 accumulation.
//              No atomics: the results are the same bits on every run.
//
// For n <= NB the whole matrix is one panel (Gauss-Jordan: the panel is all of [A | I]), so every output is the reference's bits.
// For n > NB the trailing updates sum each NB-wide block of products before subtracting it, so results agree with the reference to
// rounding, and a pivot or status decision can differ only where the deciding value lies within rounding of a tie or a threshold.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>

#include "zb_internal.h"

namespace zb {

namespace {

namespace cg = cooperative_groups;

constexpr int NB = 64;            // panel width
constexpr int PANEL_THREADS = 256;
constexpr int MIN_PANEL_ROWS = 32;  // rows per panel CTA below which another CTA costs more in the barrier than it saves

template <typename T> struct Eps;
template <> struct Eps<float> { static constexpr float v = 1.1920928955078125e-07f; };   // std.math.floatEps(f32) = 2^-23
template <> struct Eps<double> { static constexpr double v = 2.220446049250313e-16; };   // 2^-52

enum : int { ST_OK = 0, ST_SINGULAR = 1, ST_NOT_PD = 2 };

// ------------------------------------------------------------------------------------------------------------------------------
// Panel: unblocked LU (rows k0..n-1) or Gauss-Jordan (rows 0..n-1) of `width` columns starting at column k0, factoring the first
// nf of them.  Row r of the slab is matrix row row0 + r.
template <typename T>
struct PanelArgs {
    T* a;
    size_t lda;
    int row0, rows, k0, width, nf, rows_per_cta;
    int* ipiv;          // ipiv[k] = the row swapped with row k (global)
    T* cand;            // [2][grid][width] each CTA's candidate pivot row
    T* cand_key;        // [2][grid] its |value| (-1: none / NaN)
    int* cand_row;      // [2][grid] its slab row
    T* diag_row;        // [2][width] slab row k before the swap
    int* status;
};

template <typename T>
__device__ __forceinline__ void better(T& key, int& row, T k2, int r2) {
    if (k2 > key || (k2 == key && r2 < row)) { key = k2; row = r2; }
}

template <typename T, bool GJ>
__global__ void __launch_bounds__(PANEL_THREADS) panel_kernel(PanelArgs<T> p) {
    cg::grid_group grid = cg::this_grid();
    extern __shared__ __align__(16) unsigned char panel_smem[];
    const int W = p.width;
    T* S = reinterpret_cast<T*>(panel_smem);                 // [rows_per_cta][W]
    T* P = S + (size_t)p.rows_per_cta * W;                   // [W] pivot row
    __shared__ T red_key[PANEL_THREADS / 32];
    __shared__ int red_row[PANEL_THREADS / 32];
    __shared__ int s_piv;
    const int tid = threadIdx.x, b = blockIdx.x, G = gridDim.x;
    const int r_lo = b * p.rows_per_cta, r_hi = min(p.rows, r_lo + p.rows_per_cta), my = max(0, r_hi - r_lo);
    if (*p.status) return;   // an earlier panel already failed (uniform: read before any barrier)
    for (int e = tid; e < my * W; e += PANEL_THREADS) {
        const int r = e / W, j = e - r * W;
        S[e] = p.a[(size_t)(p.row0 + r_lo + r) * p.lda + p.k0 + j];
    }
    __syncthreads();
    for (int c = 0; c < p.nf; ++c) {
        const int par = c & 1;
        const int kl = p.k0 + c - p.row0;   // slab row of the pivot position
        // 1. this CTA's first maximal |a[r][c]| over its rows r >= kl (NaN never wins)
        T key = (T)-1;
        int row = 0x7fffffff;
        for (int r = max(kl, r_lo) + tid; r < r_hi; r += PANEL_THREADS) {
            const T v = S[(size_t)(r - r_lo) * W + c];
            better(key, row, isnan(v) ? (T)-1 : (T)fabs(v), r);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const T k2 = __shfl_down_sync(0xffffffffu, key, o);
            const int r2 = __shfl_down_sync(0xffffffffu, row, o);
            better(key, row, k2, r2);
        }
        if ((tid & 31) == 0) { red_key[tid >> 5] = key; red_row[tid >> 5] = row; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < PANEL_THREADS / 32; ++w) better(key, row, red_key[w], red_row[w]);
            p.cand_key[par * G + b] = key;
            p.cand_row[par * G + b] = row;
            s_piv = row;
        }
        __syncthreads();
        // 2. publish the candidate row and (owner only) the row at the pivot position
        const int cr = s_piv;
        if (cr != 0x7fffffff)
            for (int j = tid; j < W; j += PANEL_THREADS) p.cand[((size_t)par * G + b) * W + j] = S[(size_t)(cr - r_lo) * W + j];
        if (kl >= r_lo && kl < r_hi)
            for (int j = tid; j < W; j += PANEL_THREADS) p.diag_row[(size_t)par * W + j] = S[(size_t)(kl - r_lo) * W + j];
        grid.sync();
        // 3. every CTA: the same winner from the same published data
        if (tid == 0) {
            T bk = (T)-1;
            int br = 0x7fffffff, bb = -1;
            for (int q = 0; q < G; ++q) {
                const T k2 = p.cand_key[par * G + q];
                const int r2 = p.cand_row[par * G + q];
                if (k2 > bk || (k2 == bk && r2 < br)) { bk = k2; br = r2; bb = q; }
            }
            const T d = p.diag_row[(size_t)par * W + c];
            if (isnan(d)) { br = kl; bb = -1; }    // the scan starts at the diagonal, and nothing compares greater than NaN
            if (br == kl) bb = -1;
            if constexpr (GJ) {
                const T maxv = bb < 0 ? (T)fabs(d) : bk;
                if (maxv < Eps<T>::v * (T)10) {     // Matrix.zig:543
                    if (b == 0) *p.status = ST_SINGULAR;
                    br = -1;
                }
            }
            if (b == 0 && br >= 0) p.ipiv[p.k0 + c] = p.row0 + br;
            s_piv = br;
            red_row[0] = bb;
        }
        __syncthreads();
        const int pr = s_piv, pb = red_row[0];
        if (pr < 0) return;   // Singular: uniform across the grid
        const T* src = pb < 0 ? p.diag_row + (size_t)par * W : p.cand + ((size_t)par * G + pb) * W;
        for (int j = tid; j < W; j += PANEL_THREADS) P[j] = src[j];
        __syncthreads();
        // 4. the interchange
        if (pr != kl) {
            if (kl >= r_lo && kl < r_hi)
                for (int j = tid; j < W; j += PANEL_THREADS) S[(size_t)(kl - r_lo) * W + j] = P[j];
            if (pr >= r_lo && pr < r_hi)
                for (int j = tid; j < W; j += PANEL_THREADS) S[(size_t)(pr - r_lo) * W + j] = p.diag_row[(size_t)par * W + j];
        }
        __syncthreads();
        // 5. elimination
        const T piv = P[c];
        if constexpr (!GJ) {
            // Matrix.zig:1298-1306: factor = a[i][c] / pivot, a[i][j] -= factor * a[k][j]; a small pivot leaves a zero L column
            const bool elim = fabs(piv) > Eps<T>::v;
            const int i0 = max(kl + 1, r_lo);
            for (int r = i0 + tid; r < r_hi; r += PANEL_THREADS) {
                T& x = S[(size_t)(r - r_lo) * W + c];
                x = elim ? x / piv : (T)0;
            }
            __syncthreads();
            if (elim) {
                const int nc = W - c - 1;
                for (int e = tid; e < max(0, r_hi - i0) * nc; e += PANEL_THREADS) {
                    const int r = i0 + e / nc, j = c + 1 + e % nc;
                    T* row = S + (size_t)(r - r_lo) * W;
                    const T prod = row[c] * P[j];
                    row[j] = row[j] - prod;
                }
            }
        } else {
            // Matrix.zig:557-570: the pivot row divided by the pivot, every other row eliminated.  Column c keeps the pivot (pivot row)
            // or the factor (other rows): the block-row and update steps read them from there.
            __syncthreads();   // every thread holds piv before P[c] is overwritten
            for (int j = c + tid; j < W; j += PANEL_THREADS) P[j] = P[j] / piv;
            __syncthreads();
            if (kl >= r_lo && kl < r_hi) {
                T* row = S + (size_t)(kl - r_lo) * W;
                for (int j = c + 1 + tid; j < W; j += PANEL_THREADS) row[j] = P[j];
                if (tid == 0) row[c] = piv;
            }
            const int nc = W - c - 1;
            for (int e = tid; e < my * nc; e += PANEL_THREADS) {
                const int r = r_lo + e / nc, j = c + 1 + e % nc;
                if (r == kl) continue;
                T* row = S + (size_t)(r - r_lo) * W;
                const T prod = row[c] * P[j];
                row[j] = row[j] - prod;
            }
        }
        __syncthreads();
    }
    for (int e = tid; e < my * W; e += PANEL_THREADS) {
        const int r = e / W, j = e - r * W;
        p.a[(size_t)(p.row0 + r_lo + r) * p.lda + p.k0 + j] = S[e];
    }
}

template <typename T, bool GJ>
int launch_panel(T* a, size_t lda, int row0, int rows, int k0, int width, int nf, int* ipiv, T* slots, int* status, cudaStream_t s) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    auto kern = panel_kernel<T, GJ>;
    int g = std::max(1, std::min(di.sm_count, (rows + MIN_PANEL_ROWS - 1) / MIN_PANEL_ROWS));
    int rpc = (rows + g - 1) / g;
    g = (rows + rpc - 1) / rpc;
    const size_t smem = ((size_t)rpc * width + width) * sizeof(T);
    // the limit is set to the device's maximum, the same value from every call: calls on other host threads may launch concurrently
    cudaFuncAttributes fa;
    ZB_CUDA(cudaFuncGetAttributes(&fa, kern));
    const size_t smem_max = di.smem_optin - fa.sharedSizeBytes;
    if (smem > smem_max) return ZB_ERR_UNSUPPORTED;
    ZB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    int per_sm = 0;
    ZB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, PANEL_THREADS, smem));
    if (per_sm * di.sm_count < g) return ZB_ERR_UNSUPPORTED;
    // slots: [2][sm_count][NB * 2] candidate rows, then keys, then diag rows, then rows (see panel_scratch)
    PanelArgs<T> p;
    p.a = a; p.lda = lda; p.row0 = row0; p.rows = rows; p.k0 = k0; p.width = width; p.nf = nf; p.rows_per_cta = rpc;
    p.ipiv = ipiv; p.status = status;
    const size_t wmax = 2 * NB;
    p.cand = slots;
    p.cand_key = slots + 2 * (size_t)di.sm_count * wmax;
    p.diag_row = p.cand_key + 2 * (size_t)di.sm_count;
    p.cand_row = reinterpret_cast<int*>(p.diag_row + 2 * wmax);
    void* args[] = {&p};
    ZB_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(g), dim3(PANEL_THREADS), args, smem, s));
    ZB_LAUNCHED();
    return ZB_OK;
}

template <typename T>
size_t panel_scratch_bytes(int sm_count) {
    return (2 * (size_t)sm_count * 2 * NB + 2 * (size_t)sm_count + 2 * 2 * NB) * sizeof(T) + 2 * (size_t)sm_count * sizeof(int);
}

// ------------------------------------------------------------------------------------------------------------------------------
// Row interchanges ipiv[k0 .. k0+w) applied in order to every column of [0, ncols) outside [k0, k0+w).
template <typename T>
__global__ void __launch_bounds__(256) swap_kernel(T* __restrict__ a, size_t lda, int ncols, int k0, int w, const int* __restrict__ ipiv,
                                                   const int* __restrict__ status) {
    if (*status) return;
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ncols - w) return;
    if (j >= k0) j += w;
    for (int c = 0; c < w; ++c) {
        const int pr = ipiv[k0 + c];
        if (pr != k0 + c) {
            T* x = a + (size_t)(k0 + c) * lda + j;
            T* y = a + (size_t)pr * lda + j;
            const T t = *x; *x = *y; *y = t;
        }
    }
}

// LU: U12 = L11^-1 A12 for columns [j0, ncols), rows k0..k0+w-1 (Matrix.zig:1298-1306 applied to those rows: a[i][j] -= l[i][p] * a[p][j]
// in order of p, skipped where pivot p was not above eps).
template <typename T>
__global__ void __launch_bounds__(128) lu_block_row_kernel(T* __restrict__ a, size_t lda, int k0, int w, int j0, int ncols) {
    __shared__ T L[NB][NB + 1];
    __shared__ bool elim[NB];
    for (int e = threadIdx.x; e < w * w; e += blockDim.x) L[e / w][e % w] = a[(size_t)(k0 + e / w) * lda + k0 + e % w];
    __syncthreads();
    if (threadIdx.x < w) elim[threadIdx.x] = fabs(L[threadIdx.x][threadIdx.x]) > Eps<T>::v;
    __syncthreads();
    const int j = j0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ncols) return;
    T* col = a + (size_t)k0 * lda + j;
    for (int q = 0; q < w; ++q) {
        if (!elim[q]) continue;
        const T u = col[(size_t)q * lda];
        for (int i = q + 1; i < w; ++i) {
            const T prod = L[i][q] * u;
            col[(size_t)i * lda] = col[(size_t)i * lda] - prod;
        }
    }
}

// Gauss-Jordan: the block rows k0..k0+w-1 of every column j in [j0, ncols): in order of step q, row q divided by its pivot (kept at
// a[k0+q][k0+q] by the panel) and recorded in R, then every other block row i minus (its factor, a[k0+i][k0+q]) * row q.
template <typename T>
__global__ void __launch_bounds__(128) gj_block_row_kernel(T* __restrict__ a, size_t lda, int k0, int w, int j0, int ncols, T* __restrict__ R,
                                                           size_t ldr, const int* __restrict__ status) {
    if (*status) return;
    __shared__ T F[NB][NB + 1];
    for (int e = threadIdx.x; e < w * w; e += blockDim.x) F[e / w][e % w] = a[(size_t)(k0 + e / w) * lda + k0 + e % w];
    __syncthreads();
    const int j = j0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ncols) return;
    T* col = a + (size_t)k0 * lda + j;
    for (int q = 0; q < w; ++q) {
        const T v = col[(size_t)q * lda] / F[q][q];
        col[(size_t)q * lda] = v;
        R[(size_t)q * ldr + j] = v;
        for (int i = 0; i < w; ++i) {
            if (i == q) continue;
            const T prod = F[i][q] * v;
            col[(size_t)i * lda] = col[(size_t)i * lda] - prod;
        }
    }
}

// Cholesky: the w x w diagonal block at k0, left-looking (Matrix.zig:71-85 restricted to the block; one CTA).
template <typename T>
__global__ void __launch_bounds__(NB) chol_diag_kernel(T* __restrict__ a, size_t lda, int k0, int w, int* __restrict__ status) {
    if (*status) return;
    __shared__ T S[NB][NB + 1];
    __shared__ bool s_fail;
    const int t = threadIdx.x;
    for (int e = t; e < w * w; e += blockDim.x) S[e / w][e % w] = a[(size_t)(k0 + e / w) * lda + k0 + e % w];
    __syncthreads();
    for (int j = 0; j < w; ++j) {
        if (t == 0) {
            T sum = S[j][j];
            for (int k = 0; k < j; ++k) { const T prod = S[j][k] * S[j][k]; sum = sum - prod; }
            s_fail = sum <= (T)0;   // a NaN sum passes, as in the reference
            if (s_fail) *status = ST_NOT_PD;
            S[j][j] = (T)sqrt(sum);
        }
        __syncthreads();
        if (s_fail) return;
        const T ljj = S[j][j];
        for (int i = j + 1 + t; i < w; i += blockDim.x) {
            T s = S[i][j];
            for (int k = 0; k < j; ++k) { const T prod = S[i][k] * S[j][k]; s = s - prod; }
            S[i][j] = s / ljj;
        }
        __syncthreads();
    }
    for (int e = t; e < w * w; e += blockDim.x)
        if (e % w <= e / w) a[(size_t)(k0 + e / w) * lda + k0 + e % w] = S[e / w][e % w];
}

// Cholesky: L21 = A21 L11^-T, one thread per row i in [i0, n): l[i][j] = (a[i][j] - sum_k<j l[i][k] l[j][k]) / l[j][j].
template <typename T>
__global__ void __launch_bounds__(128) chol_block_col_kernel(T* __restrict__ a, size_t lda, int k0, int w, int i0, int n,
                                                             const int* __restrict__ status) {
    if (*status) return;
    __shared__ T L[NB][NB + 1];
    for (int e = threadIdx.x; e < w * w; e += blockDim.x) L[e / w][e % w] = a[(size_t)(k0 + e / w) * lda + k0 + e % w];
    __syncthreads();
    const int i = i0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    T* row = a + (size_t)i * lda + k0;
    for (int j = 0; j < w; ++j) {
        T s = row[j];
        for (int k = 0; k < j; ++k) { const T prod = row[k] * L[j][k]; s = s - prod; }
        row[j] = s / L[j][j];
    }
}

// ------------------------------------------------------------------------------------------------------------------------------
// Update: C[M x N] -= A[M x K] B[K x N]  (B element (k, j) at b[j * ldb + k] when tb).  lower: skip tiles strictly above the diagonal.
constexpr int UT = 64, UK = 16;

__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
        "{%0,%1,%2,%3};"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
          "d"(b[3]));
}

template <typename T>
__device__ __forceinline__ void load_tiles(T (*As)[UK + 1], T (*Bs)[UT + 1], const T* __restrict__ A, size_t lda, const T* __restrict__ B,
                                           size_t ldb, bool tb, int M, int N, int K, int m0, int n0, int k0, int tid, int nthreads) {
    for (int e = tid; e < UT * UK; e += nthreads) {
        const int r = e / UK, k = e % UK;
        As[r][k] = (m0 + r < M && k0 + k < K) ? A[(size_t)(m0 + r) * lda + k0 + k] : (T)0;
    }
    for (int e = tid; e < UT * UK; e += nthreads) {
        int k, c;
        if (tb) { c = e / UK; k = e % UK; } else { k = e / UT; c = e % UT; }
        Bs[k][c] = (n0 + c < N && k0 + k < K) ? (tb ? B[(size_t)(n0 + c) * ldb + k0 + k] : B[(size_t)(k0 + k) * ldb + n0 + c]) : (T)0;
    }
}

__global__ void __launch_bounds__(128) update_f64_kernel(const double* __restrict__ A, size_t lda, const double* __restrict__ B, size_t ldb,
                                                         int tb, double* __restrict__ C, size_t ldc, int M, int N, int K, int lower,
                                                         const int* __restrict__ status) {
    if (*status) return;
    const int m0 = blockIdx.y * UT, n0 = blockIdx.x * UT;
    if (lower && n0 > m0 + UT - 1) return;
    __shared__ double As[UT][UK + 1];
    __shared__ double Bs[UK][UT + 1];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    double acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.0;
    for (int k0 = 0; k0 < K; k0 += UK) {
        load_tiles<double>(As, Bs, A, lda, B, ldb, tb != 0, M, N, K, m0, n0, k0, tid, 128);
        __syncthreads();
        double af[2][8], bf[4][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int i = 0; i < 8; ++i) af[mi][i] = As[wm + 16 * mi + g + 8 * (i & 1)][t + 4 * (i >> 1)];
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int i = 0; i < 4; ++i) bf[ni][i] = Bs[t + 4 * i][wn + 8 * ni + g];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) dmma16816(acc[mi][ni], af[mi], bf[ni]);
        __syncthreads();
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int r = m0 + wm + 16 * mi + g + 8 * (q >> 1), c = n0 + wn + 8 * ni + 2 * t + (q & 1);
                if (r < M && c < N) C[(size_t)r * ldc + c] -= acc[mi][ni][q];
            }
}

__global__ void __launch_bounds__(256) update_f32_kernel(const float* __restrict__ A, size_t lda, const float* __restrict__ B, size_t ldb,
                                                         int tb, float* __restrict__ C, size_t ldc, int M, int N, int K, int lower,
                                                         const int* __restrict__ status) {
    if (*status) return;
    const int m0 = blockIdx.y * UT, n0 = blockIdx.x * UT;
    if (lower && n0 > m0 + UT - 1) return;
    __shared__ float As[UT][UK + 1];
    __shared__ float Bs[UK][UT + 1];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += UK) {
        load_tiles<float>(As, Bs, A, lda, B, ldb, tb != 0, M, N, K, m0, n0, k0, tid, 256);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < UK; ++k) {
            float av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = As[ty + 16 * i][k];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = m0 + ty + 16 * i, c = n0 + tx + 16 * j;
            if (r < M && c < N) C[(size_t)r * ldc + c] -= acc[i][j];
        }
}

template <typename T>
int update(const T* A, size_t lda, const T* B, size_t ldb, bool tb, T* C, size_t ldc, int M, int N, int K, bool lower, const int* status,
           cudaStream_t s) {
    if (M <= 0 || N <= 0 || K <= 0) return ZB_OK;
    if ((M + UT - 1) / UT > 65535) return ZB_ERR_UNSUPPORTED;
    const dim3 grid(div_up(N, UT), div_up(M, UT));
    if constexpr (sizeof(T) == 8) update_f64_kernel<<<grid, 128, 0, s>>>(A, lda, B, ldb, tb, C, ldc, M, N, K, lower, status);
    else update_f32_kernel<<<grid, 256, 0, s>>>(A, lda, B, ldb, tb, C, ldc, M, N, K, lower, status);
    ZB_LAUNCHED();
    return ZB_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// perm and sign from the interchanges (Matrix.zig:1276-1280); det = sign * u_00 * u_11 * ... in index order (:1360-1361).
template <typename T>
__global__ void perm_kernel(const int* __restrict__ ipiv, int n, uint32_t* __restrict__ perm, T* __restrict__ sign_out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    for (int i = 0; i < n; ++i) perm[i] = (uint32_t)i;
    T sign = (T)1;
    for (int k = 0; k < n; ++k) {
        const int pr = ipiv[k];
        if (pr != k) {
            sign = -sign;
            const uint32_t t = perm[k]; perm[k] = perm[pr]; perm[pr] = t;
        }
    }
    *sign_out = sign;
}

template <typename T>
__global__ void det_lu_kernel(const T* __restrict__ lu, int n, const T* __restrict__ sign, T* __restrict__ out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    T d = *sign;
    for (int i = 0; i < n; ++i) d = d * lu[(size_t)i * n + i];
    *out = d;
}

// The closed forms for n <= 3 (Matrix.zig:1345-1353), evaluated left to right (the library builds with -fmad=false: no contraction).
template <typename T>
__global__ void det_small_kernel(const T* __restrict__ a, int n, T* __restrict__ out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    auto m = [&](int i, int j) { return a[i * n + j]; };
    T d;
    if (n == 1) d = m(0, 0);
    else if (n == 2) d = m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0);
    else
        d = m(0, 0) * m(1, 1) * m(2, 2) + m(0, 1) * m(1, 2) * m(2, 0) + m(0, 2) * m(1, 0) * m(2, 1) - m(0, 2) * m(1, 1) * m(2, 0) -
            m(0, 1) * m(1, 0) * m(2, 2) - m(0, 0) * m(1, 2) * m(2, 1);
    *out = d;
}

// Matrix.inv's closed forms for n <= 3 (Matrix.zig:382-422).
template <typename T>
__global__ void inv_small_kernel(const T* __restrict__ a, int n, T* __restrict__ out, int* __restrict__ status) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    auto m = [&](int i, int j) { return a[i * n + j]; };
    const T eps = Eps<T>::v;
    if (n == 1) {
        const T d = m(0, 0);
        if (fabs(d) < eps) { *status = ST_SINGULAR; return; }
        out[0] = (T)1 / d;
    } else if (n == 2) {
        const T d = m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0);
        if (fabs(d) < eps) { *status = ST_SINGULAR; return; }
        const T r00 = m(1, 1) / d, r01 = -m(0, 1) / d, r10 = -m(1, 0) / d, r11 = m(0, 0) / d;
        out[0] = r00; out[1] = r01; out[2] = r10; out[3] = r11;
    } else {
        const T c00 = m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1);
        const T c01 = m(0, 2) * m(2, 1) - m(0, 1) * m(2, 2);
        const T c02 = m(0, 1) * m(1, 2) - m(0, 2) * m(1, 1);
        const T d = m(0, 0) * c00 + m(1, 0) * c01 + m(2, 0) * c02;
        if (fabs(d) < eps) { *status = ST_SINGULAR; return; }
        T r[9];
        r[0] = c00 / d;
        r[1] = c01 / d;
        r[2] = c02 / d;
        r[3] = (m(1, 2) * m(2, 0) - m(1, 0) * m(2, 2)) / d;
        r[4] = (m(0, 0) * m(2, 2) - m(0, 2) * m(2, 0)) / d;
        r[5] = (m(0, 2) * m(1, 0) - m(0, 0) * m(1, 2)) / d;
        r[6] = (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0)) / d;
        r[7] = (m(0, 1) * m(2, 0) - m(0, 0) * m(2, 1)) / d;
        r[8] = (m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0)) / d;
        for (int i = 0; i < 9; ++i) out[i] = r[i];
    }
}

// [A | I] (n x 2n) from A; and the right half back out.
template <typename T>
__global__ void __launch_bounds__(256) augment_kernel(const T* __restrict__ a, int n, T* __restrict__ g) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)n * 2 * n) return;
    const size_t i = e / (2 * (size_t)n), j = e % (2 * (size_t)n);
    g[e] = j < (size_t)n ? a[i * n + j] : (j - n == i ? (T)1 : (T)0);
}
template <typename T>
__global__ void __launch_bounds__(256) right_half_kernel(const T* __restrict__ g, int n, T* __restrict__ out) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)n * n) return;
    out[e] = g[(e / n) * 2 * n + n + e % n];
}

// The strict upper triangle of chol's result is zero (Matrix.zig:1328-1330).
template <typename T>
__global__ void __launch_bounds__(256) zero_upper_kernel(T* __restrict__ a, int n, const int* __restrict__ status) {
    if (*status) return;
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)n * n) return;
    if (e % n > e / n) a[e] = (T)0;
}

// ------------------------------------------------------------------------------------------------------------------------------
// LuResult.solve's scale: u_max = max |U| over the upper triangle (@max ignores NaN, as fmax does), then Singular when u_max == 0 or a
// pivot |u_ii| < u_max * eps * 100 (Matrix.zig:1200-1212).
template <typename T>
__global__ void __launch_bounds__(256) umax_kernel(const T* __restrict__ lu, int n, T* __restrict__ partial) {
    T m = (T)0;
    for (int i = blockIdx.x; i < n; i += gridDim.x)
        for (int j = i + threadIdx.x; j < n; j += blockDim.x) m = fmax(m, (T)fabs(lu[(size_t)i * n + j]));
    __shared__ T red[256];
    red[threadIdx.x] = m;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}
template <typename T>
__global__ void __launch_bounds__(256) pivot_check_kernel(const T* __restrict__ lu, int n, const T* __restrict__ partial, int parts,
                                                          int* __restrict__ status) {
    __shared__ T s_max;
    __shared__ int s_bad;
    if (threadIdx.x == 0) {
        T m = (T)0;
        for (int q = 0; q < parts; ++q) m = fmax(m, partial[q]);
        s_max = m;
        s_bad = m == (T)0;
    }
    __syncthreads();
    const T tol = s_max * Eps<T>::v * (T)100;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (fabs(lu[(size_t)i * n + i]) < tol) s_bad = 1;
    __syncthreads();
    if (threadIdx.x == 0 && s_bad) *status = ST_SINGULAR;
}

template <typename T>
__global__ void __launch_bounds__(256) gather_rows_kernel(const T* __restrict__ b, const uint32_t* __restrict__ perm, int n, int k,
                                                          T* __restrict__ x) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)n * k) return;
    x[e] = b[(size_t)perm[e / k] * k + e % k];
}

// Diagonal-block solves of LuResult.solve, one thread per right-hand side column: forward with the unit L (:1191-1196), or backward
// with U and the division last (:1208-1218), in the reference's order inside the block.
template <typename T, bool FORWARD>
__global__ void __launch_bounds__(128) trsv_block_kernel(const T* __restrict__ lu, int n, int k0, int w, T* __restrict__ x, int k,
                                                         const int* __restrict__ status) {
    if (*status) return;
    __shared__ T D[NB][NB + 1];
    for (int e = threadIdx.x; e < w * w; e += blockDim.x) D[e / w][e % w] = lu[(size_t)(k0 + e / w) * n + k0 + e % w];
    __syncthreads();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= k) return;
    T* col = x + (size_t)k0 * k + c;
    if constexpr (FORWARD) {
        for (int i = 1; i < w; ++i) {
            T v = col[(size_t)i * k];
            for (int j = 0; j < i; ++j) { const T prod = D[i][j] * col[(size_t)j * k]; v = v - prod; }
            col[(size_t)i * k] = v;
        }
    } else {
        for (int i = w - 1; i >= 0; --i) {
            T v = col[(size_t)i * k];
            for (int j = i + 1; j < w; ++j) { const T prod = D[i][j] * col[(size_t)j * k]; v = v - prod; }
            col[(size_t)i * k] = v / D[i][i];
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------------------
struct Work {
    Scratch buf;
    int* status = nullptr;
    int* ipiv = nullptr;
    void* slots = nullptr;
    void* scalars = nullptr;   // [4] T
    int alloc(size_t n, size_t slot_bytes, cudaStream_t s) {
        const size_t ipiv_bytes = ((n * sizeof(int)) + 255) & ~(size_t)255;
        int rc = buf.alloc(256 + 256 + ipiv_bytes + slot_bytes, s);
        if (rc) return rc;
        char* p = (char*)buf.p;
        status = (int*)p;
        scalars = p + 256;
        ipiv = (int*)(p + 512);
        slots = p + 512 + ipiv_bytes;
        ZB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), s));
        return ZB_OK;
    }
};

int finish(const int* d_status, cudaStream_t s, int* st) {
    ZB_CUDA(cudaMemcpyAsync(st, d_status, sizeof(int), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    return ZB_OK;
}

// Packed LU of the n x n matrix in `a` (in place); ipiv in w.
template <typename T>
int lu_inplace(T* a, int n, Work& w, cudaStream_t s) {
    int rc;
    for (int k0 = 0; k0 < n; k0 += NB) {
        const int bw = std::min(NB, n - k0);
        if ((rc = launch_panel<T, false>(a, n, k0, n - k0, k0, bw, bw, w.ipiv, (T*)w.slots, w.status, s))) return rc;
        if (n > bw) {
            swap_kernel<T><<<div_up(n - bw, 256), 256, 0, s>>>(a, n, n, k0, bw, w.ipiv, w.status);
            ZB_LAUNCHED();
        }
        const int j0 = k0 + bw;
        if (j0 < n) {
            lu_block_row_kernel<T><<<div_up(n - j0, 128), 128, 0, s>>>(a, n, k0, bw, j0, n);
            ZB_LAUNCHED();
            const size_t ld = n;
            if ((rc = update<T>(a + (size_t)j0 * ld + k0, ld, a + (size_t)k0 * ld + j0, ld, false, a + (size_t)j0 * ld + j0, ld, n - j0, n - j0,
                                bw, false, w.status, s)))
                return rc;
        }
    }
    return ZB_OK;
}

template <typename T>
int work_for(Work& w, int n, cudaStream_t s) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    return w.alloc((size_t)n, panel_scratch_bytes<T>(di.sm_count), s);
}

int status_code(int st) { return st == ST_SINGULAR ? ZB_ERR_SINGULAR : st == ST_NOT_PD ? ZB_ERR_NOT_POSITIVE_DEFINITE : ZB_OK; }

template <typename T>
int lu_device(const T* a, uint32_t rows, uint32_t cols, T* lu, uint32_t* perm, T* sign, cudaStream_t s) {
    if (rows != cols) return ZB_ERR_NOT_SQUARE;
    if (!sign || (rows > 0 && (!a || !lu || !perm))) return ZB_ERR_INVALID_ARGUMENT;
    if (rows > 0x7fffffffu) return ZB_ERR_UNSUPPORTED;
    const int n = (int)rows;
    if (n == 0) { *sign = (T)1; return ZB_OK; }
    Work w;
    int rc = work_for<T>(w, n, s);
    if (rc) return rc;
    if (lu != a) ZB_CUDA(cudaMemcpyAsync(lu, a, (size_t)n * n * sizeof(T), cudaMemcpyDeviceToDevice, s));
    if ((rc = lu_inplace<T>(lu, n, w, s))) return rc;
    perm_kernel<T><<<1, 1, 0, s>>>(w.ipiv, n, perm, (T*)w.scalars);
    ZB_LAUNCHED();
    ZB_CUDA(cudaMemcpyAsync(sign, w.scalars, sizeof(T), cudaMemcpyDeviceToHost, s));
    int st = 0;
    if ((rc = finish(w.status, s, &st))) return rc;
    t_last_kernel = "lu_panel";
    return status_code(st);
}

template <typename T>
int lu_solve_device(const T* lu, const uint32_t* perm, uint32_t n_, const T* b, uint32_t b_rows, uint32_t k_, T* x, cudaStream_t s) {
    if (b_rows != n_) return ZB_ERR_DIMENSION_MISMATCH;
    if (n_ == 0) return ZB_ERR_SINGULAR;   // u_max == 0 (Matrix.zig:1204)
    if (!lu || !perm || (k_ > 0 && (!b || !x))) return ZB_ERR_INVALID_ARGUMENT;
    if (n_ > 0x7fffffffu || k_ > 0x7fffffffu) return ZB_ERR_UNSUPPORTED;
    const int n = (int)n_, k = (int)k_;
    Work w;
    int rc = w.alloc(0, 1024 * sizeof(T), s);
    if (rc) return rc;
    if (k > 0) {
        gather_rows_kernel<T><<<div_up((size_t)n * k, 256), 256, 0, s>>>(b, perm, n, k, x);
        ZB_LAUNCHED();
        for (int k0 = 0; k0 < n; k0 += NB) {
            const int bw = std::min(NB, n - k0);
            trsv_block_kernel<T, true><<<div_up(k, 128), 128, 0, s>>>(lu, n, k0, bw, x, k, w.status);
            ZB_LAUNCHED();
            if ((rc = update<T>(lu + (size_t)(k0 + bw) * n + k0, n, x + (size_t)k0 * k, k, false, x + (size_t)(k0 + bw) * k, k, n - k0 - bw, k,
                                bw, false, w.status, s)))
                return rc;
        }
    }
    const int parts = std::min(1024, n);
    umax_kernel<T><<<parts, 256, 0, s>>>(lu, n, (T*)w.slots);
    ZB_LAUNCHED();
    pivot_check_kernel<T><<<1, 256, 0, s>>>(lu, n, (T*)w.slots, parts, w.status);
    ZB_LAUNCHED();
    if (k > 0) {
        for (int k0 = ((n - 1) / NB) * NB; k0 >= 0; k0 -= NB) {
            const int bw = std::min(NB, n - k0);
            trsv_block_kernel<T, false><<<div_up(k, 128), 128, 0, s>>>(lu, n, k0, bw, x, k, w.status);
            ZB_LAUNCHED();
            if ((rc = update<T>(lu + k0, n, x + (size_t)k0 * k, k, false, x, k, k0, k, bw, false, w.status, s))) return rc;
        }
    }
    int st = 0;
    if ((rc = finish(w.status, s, &st))) return rc;
    t_last_kernel = "lu_solve_trsv";
    return status_code(st);
}

template <typename T>
int det_device(const T* a, uint32_t rows, uint32_t cols, T* det, cudaStream_t s) {
    if (rows != cols) return ZB_ERR_NOT_SQUARE;
    if (rows == 0) return ZB_ERR_DIMENSION_MISMATCH;
    if (!a || !det) return ZB_ERR_INVALID_ARGUMENT;
    if (rows > 0x7fffffffu) return ZB_ERR_UNSUPPORTED;
    const int n = (int)rows;
    Work w;
    int rc = work_for<T>(w, n, s);
    if (rc) return rc;
    T* d_out = (T*)w.scalars + 1;
    Scratch luw;
    if (n <= 3) {
        det_small_kernel<T><<<1, 1, 0, s>>>(a, n, d_out);
        ZB_LAUNCHED();
    } else {
        if ((rc = luw.alloc((size_t)n * n * sizeof(T), s))) return rc;
        ZB_CUDA(cudaMemcpyAsync(luw.p, a, (size_t)n * n * sizeof(T), cudaMemcpyDeviceToDevice, s));
        if ((rc = lu_inplace<T>(luw.as<T>(), n, w, s))) return rc;
        Scratch perm;
        if ((rc = perm.alloc((size_t)n * sizeof(uint32_t), s))) return rc;
        perm_kernel<T><<<1, 1, 0, s>>>(w.ipiv, n, perm.as<uint32_t>(), (T*)w.scalars);
        ZB_LAUNCHED();
        det_lu_kernel<T><<<1, 1, 0, s>>>(luw.as<T>(), n, (T*)w.scalars, d_out);
        ZB_LAUNCHED();
    }
    ZB_CUDA(cudaMemcpyAsync(det, d_out, sizeof(T), cudaMemcpyDeviceToHost, s));
    int st = 0;
    if ((rc = finish(w.status, s, &st))) return rc;
    t_last_kernel = n <= 3 ? "det_closed_form" : "lu_panel";
    return status_code(st);
}

template <typename T>
int inv_device(const T* a, uint32_t rows, uint32_t cols, T* out, cudaStream_t s) {
    if (rows != cols) return ZB_ERR_NOT_SQUARE;
    if (rows == 0) return ZB_ERR_DIMENSION_MISMATCH;   // the reference reaches `unreachable` here
    if (!a || !out) return ZB_ERR_INVALID_ARGUMENT;
    if (rows > 0x3fffffffu) return ZB_ERR_UNSUPPORTED;
    const int n = (int)rows;
    Work w;
    int rc = work_for<T>(w, n, s);
    if (rc) return rc;
    if (n <= 3) {
        inv_small_kernel<T><<<1, 1, 0, s>>>(a, n, out, w.status);
        ZB_LAUNCHED();
    } else {
        Scratch aug;
        const size_t ld = 2 * (size_t)n;
        if ((rc = aug.alloc((size_t)n * ld * sizeof(T), s))) return rc;
        T* g = aug.as<T>();
        augment_kernel<T><<<div_up((size_t)n * ld, 256), 256, 0, s>>>(a, n, g);
        ZB_LAUNCHED();
        if (n <= NB) {
            // the whole of [A | I] is one panel: the reference's arithmetic in its order
            if ((rc = launch_panel<T, true>(g, ld, 0, n, 0, 2 * n, n, w.ipiv, (T*)w.slots, w.status, s))) return rc;
        } else {
            Scratch rbuf;
            if ((rc = rbuf.alloc((size_t)NB * ld * sizeof(T), s))) return rc;
            T* R = rbuf.as<T>();
            for (int k0 = 0; k0 < n; k0 += NB) {
                const int bw = std::min(NB, n - k0), j0 = k0 + bw;
                if ((rc = launch_panel<T, true>(g, ld, 0, n, k0, bw, bw, w.ipiv, (T*)w.slots, w.status, s))) return rc;
                swap_kernel<T><<<div_up(2 * n - bw, 256), 256, 0, s>>>(g, ld, 2 * n, k0, bw, w.ipiv, w.status);
                ZB_LAUNCHED();
                gj_block_row_kernel<T><<<div_up(2 * n - j0, 128), 128, 0, s>>>(g, ld, k0, bw, j0, 2 * n, R, ld, w.status);
                ZB_LAUNCHED();
                // every row outside the block: a[i][j] -= factor[i][q] * r_q[j] over the block's steps q
                if ((rc = update<T>(g + k0, ld, R + j0, ld, false, g + j0, ld, k0, 2 * n - j0, bw, false, w.status, s))) return rc;
                if ((rc = update<T>(g + (size_t)j0 * ld + k0, ld, R + j0, ld, false, g + (size_t)j0 * ld + j0, ld, n - j0, 2 * n - j0, bw, false,
                                    w.status, s)))
                    return rc;
            }
        }
        right_half_kernel<T><<<div_up((size_t)n * n, 256), 256, 0, s>>>(g, n, out);
        ZB_LAUNCHED();
    }
    int st = 0;
    if ((rc = finish(w.status, s, &st))) return rc;
    t_last_kernel = n <= 3 ? "inv_closed_form" : "gauss_jordan_panel";
    return status_code(st);
}

template <typename T>
int chol_device(const T* a, uint32_t rows, uint32_t cols, T* l, cudaStream_t s) {
    if (rows != cols) return ZB_ERR_NOT_SQUARE;
    if (rows > 0 && (!a || !l)) return ZB_ERR_INVALID_ARGUMENT;
    if (rows > 0x7fffffffu) return ZB_ERR_UNSUPPORTED;
    const int n = (int)rows;
    if (n == 0) return ZB_OK;
    Work w;
    int rc = w.alloc(0, 0, s);
    if (rc) return rc;
    if (l != a) ZB_CUDA(cudaMemcpyAsync(l, a, (size_t)n * n * sizeof(T), cudaMemcpyDeviceToDevice, s));
    for (int k0 = 0; k0 < n; k0 += NB) {
        const int bw = std::min(NB, n - k0), i0 = k0 + bw;
        chol_diag_kernel<T><<<1, NB, 0, s>>>(l, n, k0, bw, w.status);
        ZB_LAUNCHED();
        if (i0 < n) {
            chol_block_col_kernel<T><<<div_up(n - i0, 128), 128, 0, s>>>(l, n, k0, bw, i0, n, w.status);
            ZB_LAUNCHED();
            const T* l21 = l + (size_t)i0 * n + k0;
            if ((rc = update<T>(l21, n, l21, n, true, l + (size_t)i0 * n + i0, n, n - i0, n - i0, bw, true, w.status, s))) return rc;
        }
    }
    zero_upper_kernel<T><<<div_up((size_t)n * n, 256), 256, 0, s>>>(l, n, w.status);
    ZB_LAUNCHED();
    int st = 0;
    if ((rc = finish(w.status, s, &st))) return rc;
    t_last_kernel = "chol_panel";
    return status_code(st);
}

}  // namespace

}  // namespace zb

using namespace zb;

extern "C" {

int zb_lu_f32(const float* a, uint32_t rows, uint32_t cols, float* lu, uint32_t* perm, float* sign, zb_stream s) {
    return lu_device<float>(a, rows, cols, lu, perm, sign, (cudaStream_t)s);
}
int zb_lu_f64(const double* a, uint32_t rows, uint32_t cols, double* lu, uint32_t* perm, double* sign, zb_stream s) {
    return lu_device<double>(a, rows, cols, lu, perm, sign, (cudaStream_t)s);
}
int zb_lu_solve_f32(const float* lu, const uint32_t* perm, uint32_t n, const float* b, uint32_t b_rows, uint32_t k, float* x, zb_stream s) {
    return lu_solve_device<float>(lu, perm, n, b, b_rows, k, x, (cudaStream_t)s);
}
int zb_lu_solve_f64(const double* lu, const uint32_t* perm, uint32_t n, const double* b, uint32_t b_rows, uint32_t k, double* x, zb_stream s) {
    return lu_solve_device<double>(lu, perm, n, b, b_rows, k, x, (cudaStream_t)s);
}
int zb_det_f32(const float* a, uint32_t rows, uint32_t cols, float* det, zb_stream s) {
    return det_device<float>(a, rows, cols, det, (cudaStream_t)s);
}
int zb_det_f64(const double* a, uint32_t rows, uint32_t cols, double* det, zb_stream s) {
    return det_device<double>(a, rows, cols, det, (cudaStream_t)s);
}
int zb_inv_f32(const float* a, uint32_t rows, uint32_t cols, float* out, zb_stream s) {
    return inv_device<float>(a, rows, cols, out, (cudaStream_t)s);
}
int zb_inv_f64(const double* a, uint32_t rows, uint32_t cols, double* out, zb_stream s) {
    return inv_device<double>(a, rows, cols, out, (cudaStream_t)s);
}
int zb_chol_f32(const float* a, uint32_t rows, uint32_t cols, float* l, zb_stream s) {
    return chol_device<float>(a, rows, cols, l, (cudaStream_t)s);
}
int zb_chol_f64(const double* a, uint32_t rows, uint32_t cols, double* l, zb_stream s) {
    return chol_device<double>(a, rows, cols, l, (cudaStream_t)s);
}

}  // extern "C"
