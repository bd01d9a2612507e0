// zb_jacobi.cu -- Matrix.svd / SMatrix.svd (reference Matrix.zig:1570, SMatrix.zig:804, svd.zig:80-496) and Matrix.eigh
// (reference matrix/eigen.zig:34-136) as parallel Jacobi methods on the GPU.
//
// The reference computes the SVD with a sequential Golub-Reinsch routine (Householder bidiagonalisation + implicit-shift QR)
// and eigh with a cyclic (sequential) Jacobi sweep.  Neither maps to a GPU: every step depends on the previous one.  This file
// uses the Jacobi family in its PARALLEL ordering instead:
//
//   * SVD: one-sided (Hestenes) Jacobi.  The columns of A are rotated in pairs until they are mutually orthogonal; then
//     sigma_j = |a_j|, u_j = a_j / sigma_j, and V accumulates the rotations.  A round-robin tournament schedules n/2 disjoint
//     column pairs per round (n - 1 rounds per sweep), so a round is n/2 independent (dot products + rotation) tasks: one CTA per
//     pair, coalesced over the column length, f64 accumulation of the three dot products, and one grid-wide barrier per round
//     inside a single persistent cooperative kernel.  Converges quadratically (6-10 sweeps), and computes small singular values
//     to high RELATIVE accuracy -- better than the bidiagonalisation route.
//   * eigh: two-sided Jacobi with the same tournament: per round the n/2 rotation angles are computed from (a_pp, a_qq, a_pq),
//     then all column pairs are rotated, then all row pairs (three barriers per round); V accumulates the column rotations.
//
// Matrices of fewer than kDeviceMinN columns are done by the same algorithm on the host (a launch costs more than the whole
// decomposition); both share the rotation formulas below, so they agree to rounding.
//
// Results are defined up to the sign of each singular / eigen vector pair and the order inside a cluster of equal values, like
// any SVD; the parity criterion is the reference's own (test_svd_comparison.zig:51-72, svd.zig:498-636): singular values to
// sqrt(eps), orthonormal factors, A = U S V^T.  The one caller whose OUTPUT depends on the sign convention of the reference's
// routine, fdm (W = Us D Ut^T mixes the vectors of two different decompositions), keeps its own fixed-size 3x3 solve (zb_fdm.cu).
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <vector>

#include "zb_internal.h"

namespace zb {
namespace {

constexpr uint32_t kDeviceMinN = 24;   // below this the host runs the same algorithm
constexpr int kMaxSweeps = 60;
thread_local int t_last_sweeps = 0;    // sweeps the last decomposition on this thread needed (zb_last_sweeps)

// ---- shared rotation math ----------------------------------------------------------------------------------------
#ifdef __CUDACC__
#define ZJ_HD __host__ __device__ __forceinline__
#else
#define ZJ_HD inline
#endif

// pair k of round r of the round-robin tournament over np (even) players; returns p < q
ZJ_HD void tournament_pair(int np, int r, int k, int& p, int& q) {
    int a, b;
    if (k == 0) { a = np - 1; b = r; }
    else { a = (r + k) % (np - 1); b = (r - k + (np - 1)) % (np - 1); }
    p = a < b ? a : b;
    q = a < b ? b : a;
}

// one-sided: rotation that makes columns with norms^2 alpha, beta and inner product gamma orthogonal
template <typename T>
ZJ_HD bool hestenes_rotation(double alpha, double beta, double gamma, double tol, double abs_floor, T& c, T& s) {
    // orthogonal to working precision, or both columns are rounding noise of a rank-deficient matrix (|gamma| at the level of
    // (eps |A|)^2: rotating noise against noise would never settle)
    if (gamma == 0.0 || fabs(gamma) <= abs_floor) return false;
    // On the device a pair is one dependency chain and the f64 divisions and square roots are most of it (ncu: ~535 instructions per
    // pair and round with the textbook form zeta = (beta - alpha) / 2 gamma, t = sgn / (|zeta| + sqrt(1 + zeta^2)), c = 1 / sqrt(1 + t^2)
    // and a square root in the test: three of each).  The same rotation with one division and two square roots:
    //   t = 2 gamma sgn(d) / (|d| + sqrt(d^2 + 4 gamma^2)),  d = beta - alpha   (a sum of positives: no cancellation)
    //   c = rsqrt(1 + t^2)
    // and, for f32 data (whose squared sums stay far inside the f64 range), the test on squares.
    if (sizeof(T) == 4) {
        if (gamma * gamma <= tol * tol * alpha * beta) return false;
    } else if (fabs(gamma) <= tol * sqrt(alpha * beta)) {
        return false;
    }
    const double d = beta - alpha;
    const double t = (d >= 0.0 ? 2.0 : -2.0) * gamma / (fabs(d) + sqrt(d * d + 4.0 * gamma * gamma));
#ifdef __CUDA_ARCH__
    const double cc = rsqrt(1.0 + t * t);
#else
    const double cc = 1.0 / sqrt(1.0 + t * t);
#endif
    c = (T)cc;
    s = (T)(cc * t);
    return true;
}

// two-sided: rotation that annihilates a_pq of a symmetric matrix
template <typename T>
ZJ_HD bool symmetric_rotation(double app, double aqq, double apq, double tiny, T& c, T& s) {
    if (apq == 0.0 || fabs(apq) <= tiny) return false;
    const double theta = (aqq - app) / (2.0 * apq);
    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(1.0 + theta * theta));
    const double cc = 1.0 / sqrt(1.0 + t * t);
    c = (T)cc;
    s = (T)(cc * t);
    return true;
}

// ---- device kernels ----------------------------------------------------------------------------------------------
struct GridBarrier {
    unsigned int* counter;   // monotone
    unsigned int generation;
    __device__ void sync() {
        __syncthreads();
        if (threadIdx.x == 0) {
            ++generation;
            __threadfence();
            atomicAdd(counter, 1u);
            const unsigned int target = generation * gridDim.x;
            while (*(volatile unsigned int*)counter < target) {}
            __threadfence();
        }
        __syncthreads();
    }
};

template <int NT>
__device__ __forceinline__ void block_sum3(double& a, double& b, double& c) {
    __shared__ double red[3][NT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_down_sync(0xffffffffu, a, o);
        b += __shfl_down_sync(0xffffffffu, b, o);
        c += __shfl_down_sync(0xffffffffu, c, o);
    }
    __syncthreads();   // the previous use of `red` is over
    if (lane == 0) { red[0][warp] = a; red[1][warp] = b; red[2][warp] = c; }
    __syncthreads();
    a = b = c = 0.0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) { a += red[0][w]; b += red[1][w]; c += red[2][w]; }   // every thread: the same order
}

// Gt: n columns of A stored as rows of length m; Vt: n rows of length n (row j = column j of V).
template <typename T, int NT>
__global__ void __launch_bounds__(NT) jacobi_svd_kernel(T* __restrict__ Gt, T* __restrict__ Vt, int m, int n, int with_v, double tol, double abs_floor,
                                                        unsigned int* barrier_counter, unsigned int* rotations /* [kMaxSweeps] */,
                                                        int* sweeps_done) {
    GridBarrier bar{barrier_counter, 0};
    const int np = n + (n & 1);
    int sweep = 0;
    for (; sweep < kMaxSweeps; ++sweep) {
        for (int r = 0; r < np - 1; ++r) {
            for (int k = blockIdx.x; k < np / 2; k += gridDim.x) {
                int p, q;
                tournament_pair(np, r, k, p, q);
                if (q >= n) continue;   // the bye of an odd n
                T* gp = Gt + (size_t)p * m;
                T* gq = Gt + (size_t)q * m;
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = threadIdx.x; i < m; i += NT) {
                    const double x = (double)__ldcg(gp + i), y = (double)__ldcg(gq + i);   // other CTAs wrote these in earlier rounds: bypass L1
                    alpha += x * x;
                    beta += y * y;
                    gamma += x * y;
                }
                block_sum3<NT>(alpha, beta, gamma);
                T c, s;
                if (!hestenes_rotation<T>(alpha, beta, gamma, tol, abs_floor, c, s)) continue;   // uniform across the block
                if (threadIdx.x == 0) atomicAdd(&rotations[sweep], 1u);
                for (int i = threadIdx.x; i < m; i += NT) {
                    const T x = __ldcg(gp + i), y = __ldcg(gq + i);
                    gp[i] = c * x - s * y;
                    gq[i] = s * x + c * y;
                }
                if (with_v) {
                    T* vp = Vt + (size_t)p * n;
                    T* vq = Vt + (size_t)q * n;
                    for (int i = threadIdx.x; i < n; i += NT) {
                        const T x = __ldcg(vp + i), y = __ldcg(vq + i);
                        vp[i] = c * x - s * y;
                        vq[i] = s * x + c * y;
                    }
                }
            }
            bar.sync();
        }
        if (*(volatile unsigned int*)&rotations[sweep] == 0) break;   // a full sweep without a rotation: converged
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *sweeps_done = sweep;
}

// The same sweep with one WARP per column pair (short columns: the three dot products are 5 shuffle steps, no block barrier, and
// a quarter of the CTAs take part in the grid barrier, which is what a round costs at this size).
template <typename T, int NT>
__global__ void __launch_bounds__(NT) jacobi_svd_warp_kernel(T* __restrict__ Gt, T* __restrict__ Vt, int m, int n, int with_v, double tol,
                                                             double abs_floor, unsigned int* barrier_counter, unsigned int* rotations,
                                                             int* sweeps_done) {
    GridBarrier bar{barrier_counter, 0};
    const int np = n + (n & 1);
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * (NT / 32) + (threadIdx.x >> 5), n_warps = gridDim.x * (NT / 32);
    int sweep = 0;
    for (; sweep < kMaxSweeps; ++sweep) {
        for (int r = 0; r < np - 1; ++r) {
            for (int k = warp_global; k < np / 2; k += n_warps) {
                int p, q;
                tournament_pair(np, r, k, p, q);
                if (q >= n) continue;
                T* gp = Gt + (size_t)p * m;
                T* gq = Gt + (size_t)q * m;
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = lane; i < m; i += 32) {
                    const double x = (double)__ldcg(gp + i), y = (double)__ldcg(gq + i);
                    alpha += x * x;
                    beta += y * y;
                    gamma += x * y;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {   // xor butterfly: every lane ends with the same totals
                    alpha += __shfl_xor_sync(0xffffffffu, alpha, o);
                    beta += __shfl_xor_sync(0xffffffffu, beta, o);
                    gamma += __shfl_xor_sync(0xffffffffu, gamma, o);
                }
                T c, s;
                if (!hestenes_rotation<T>(alpha, beta, gamma, tol, abs_floor, c, s)) continue;
                if (lane == 0) atomicAdd(&rotations[sweep], 1u);
                for (int i = lane; i < m; i += 32) {
                    const T x = __ldcg(gp + i), y = __ldcg(gq + i);
                    gp[i] = c * x - s * y;
                    gq[i] = s * x + c * y;
                }
                if (with_v) {
                    T* vp = Vt + (size_t)p * n;
                    T* vq = Vt + (size_t)q * n;
                    for (int i = lane; i < n; i += 32) {
                        const T x = __ldcg(vp + i), y = __ldcg(vq + i);
                        vp[i] = c * x - s * y;
                        vq[i] = s * x + c * y;
                    }
                }
            }
            bar.sync();
        }
        if (*(volatile unsigned int*)&rotations[sweep] == 0) break;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *sweeps_done = sweep;
}

// The same sweep for matrices that fit the shared memory of ONE thread-block cluster (PCA's covariance: 256 x 256 f32 + V = 512 KB
// over 8 CTAs): the columns of A and V live in distributed shared memory, a warp rotates one pair per round reading and writing the
// two columns wherever they are (ld / st.shared::cluster through cluster.map_shared_rank), and the barrier between rounds is the
// hardware cluster barrier instead of an atomic counter in global memory.  Arithmetic, pair order and stopping rule are the warp
// kernel's (bit-identical results).  Measured on the 256 x 256 f32 covariance (8 sweeps + the closing one, 2295 rounds): 9.0 ms
// against 11.1 ms -- 3.9 us per round, now the chain inside a pair: remote loads, f64 dot products and shuffles, the f64 divisions
// and square roots of the rotation, the two updates.  (Fetching the V columns together with the A columns changed nothing.)
constexpr int kClusterCtas = 8;
constexpr int kClusterThreads = 512;

template <typename T>
__global__ void __launch_bounds__(kClusterThreads) jacobi_svd_cluster_kernel(T* __restrict__ Gt, T* __restrict__ Vt, int m, int n, int with_v, double tol,
                                                                             double abs_floor, unsigned int* rotations, int* sweeps_done) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) unsigned char jc_smem[];
    const int np = n + (n & 1);
    const int cpc = (np + kClusterCtas - 1) / kClusterCtas;        // columns per CTA
    T* g_loc = reinterpret_cast<T*>(jc_smem);                      // [cpc][m]
    T* v_loc = g_loc + (size_t)cpc * m;                            // [cpc][n]
    unsigned int* rot_loc = reinterpret_cast<unsigned int*>(v_loc + (with_v ? (size_t)cpc * n : 0));   // rotations of this CTA in the running sweep (V is only allocated when wanted)
    const unsigned rank = cluster.block_rank();
    const int lane = threadIdx.x & 31;
    const int warp_global = (int)rank * (kClusterThreads / 32) + (threadIdx.x >> 5), n_warps = kClusterCtas * (kClusterThreads / 32);
    // my columns: global -> shared
    for (int j = 0; j < cpc; ++j) {
        const int col = (int)rank * cpc + j;
        for (int i = threadIdx.x; i < m; i += kClusterThreads) g_loc[(size_t)j * m + i] = col < n ? Gt[(size_t)col * m + i] : (T)0;
        if (with_v)
            for (int i = threadIdx.x; i < n; i += kClusterThreads) v_loc[(size_t)j * n + i] = col < n ? Vt[(size_t)col * n + i] : (T)0;
    }
    if (threadIdx.x == 0) *rot_loc = 0u;
    cluster.sync();
    auto g_col = [&](int col) { return cluster.map_shared_rank(g_loc, (unsigned)(col / cpc)) + (size_t)(col % cpc) * m; };
    auto v_col = [&](int col) { return cluster.map_shared_rank(v_loc, (unsigned)(col / cpc)) + (size_t)(col % cpc) * n; };
    int sweep = 0;
    for (; sweep < kMaxSweeps; ++sweep) {
        for (int r = 0; r < np - 1; ++r) {
            for (int k = warp_global; k < np / 2; k += n_warps) {
                int p, q;
                tournament_pair(np, r, k, p, q);
                if (q >= n) continue;
                T* gp = g_col(p);
                T* gq = g_col(q);
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = lane; i < m; i += 32) {
                    const double x = (double)gp[i], y = (double)gq[i];
                    alpha += x * x;
                    beta += y * y;
                    gamma += x * y;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    alpha += __shfl_xor_sync(0xffffffffu, alpha, o);
                    beta += __shfl_xor_sync(0xffffffffu, beta, o);
                    gamma += __shfl_xor_sync(0xffffffffu, gamma, o);
                }
                T c, s;
                if (!hestenes_rotation<T>(alpha, beta, gamma, tol, abs_floor, c, s)) continue;
                if (lane == 0) atomicAdd(rot_loc, 1u);
                for (int i = lane; i < m; i += 32) {
                    const T x = gp[i], y = gq[i];
                    gp[i] = c * x - s * y;
                    gq[i] = s * x + c * y;
                }
                if (with_v) {
                    T* vp = v_col(p);
                    T* vq = v_col(q);
                    for (int i = lane; i < n; i += 32) {
                        const T x = vp[i], y = vq[i];
                        vp[i] = c * x - s * y;
                        vq[i] = s * x + c * y;
                    }
                }
            }
            cluster.sync();
        }
        // rotations of the sweep, summed over the cluster (every CTA reads all eight counters: the same decision everywhere)
        unsigned int total = 0;
        for (unsigned rk = 0; rk < (unsigned)kClusterCtas; ++rk) total += *cluster.map_shared_rank(rot_loc, rk);
        cluster.sync();
        if (threadIdx.x == 0) *rot_loc = 0u;
        if (rank == 0 && threadIdx.x == 0) rotations[sweep] = total;
        cluster.sync();
        if (total == 0) break;
    }
    // shared -> global
    for (int j = 0; j < cpc; ++j) {
        const int col = (int)rank * cpc + j;
        if (col >= n) break;
        for (int i = threadIdx.x; i < m; i += kClusterThreads) Gt[(size_t)col * m + i] = g_loc[(size_t)j * m + i];
        if (with_v)
            for (int i = threadIdx.x; i < n; i += kClusterThreads) Vt[(size_t)col * n + i] = v_loc[(size_t)j * n + i];
    }
    if (rank == 0 && threadIdx.x == 0) *sweeps_done = sweep;
}

// A: n x n symmetric, row-major (both triangles kept up to date); Vt rows = eigenvector columns; cs: n/2 rotations of the round
template <typename T, int NT>
__global__ void __launch_bounds__(NT) jacobi_eigh_kernel(T* __restrict__ A, T* __restrict__ Vt, int n, double tiny, T* __restrict__ cs,
                                                         unsigned int* barrier_counter, unsigned int* rotations, int* sweeps_done) {
    GridBarrier bar{barrier_counter, 0};
    const int np = n + (n & 1);
    const int npairs = np / 2;
    int sweep = 0;
    for (; sweep < kMaxSweeps; ++sweep) {
        for (int r = 0; r < np - 1; ++r) {
            // 1. the angles, from the matrix as it stands
            for (int k = blockIdx.x * NT + threadIdx.x; k < npairs; k += gridDim.x * NT) {
                int p, q;
                tournament_pair(np, r, k, p, q);
                T c = (T)1, s = (T)0;
                if (q < n && symmetric_rotation<T>((double)__ldcg(A + (size_t)p * n + p), (double)__ldcg(A + (size_t)q * n + q), (double)__ldcg(A + (size_t)p * n + q), tiny, c, s))
                    atomicAdd(&rotations[sweep], 1u);
                cs[2 * k] = c;
                cs[2 * k + 1] = s;
            }
            bar.sync();
            // 2. A <- A J (columns p, q of every row) and V <- V J; task = (pair, row)
            for (long long t = (long long)blockIdx.x * NT + threadIdx.x; t < (long long)npairs * n; t += (long long)gridDim.x * NT) {
                const int k = (int)(t / n), i = (int)(t - (long long)k * n);
                int p, q;
                tournament_pair(np, r, k, p, q);
                const T c = __ldcg(cs + 2 * k), s = __ldcg(cs + 2 * k + 1);
                if (q >= n || s == (T)0) continue;
                const T x = __ldcg(A + (size_t)i * n + p), y = __ldcg(A + (size_t)i * n + q);
                A[(size_t)i * n + p] = c * x - s * y;
                A[(size_t)i * n + q] = s * x + c * y;
                const T vx = __ldcg(Vt + (size_t)p * n + i), vy = __ldcg(Vt + (size_t)q * n + i);
                Vt[(size_t)p * n + i] = c * vx - s * vy;
                Vt[(size_t)q * n + i] = s * vx + c * vy;
            }
            bar.sync();
            // 3. A <- J^T A (rows p, q of every column)
            for (long long t = (long long)blockIdx.x * NT + threadIdx.x; t < (long long)npairs * n; t += (long long)gridDim.x * NT) {
                const int k = (int)(t / n), i = (int)(t - (long long)k * n);
                int p, q;
                tournament_pair(np, r, k, p, q);
                const T c = __ldcg(cs + 2 * k), s = __ldcg(cs + 2 * k + 1);
                if (q >= n || s == (T)0) continue;
                const T x = __ldcg(A + (size_t)p * n + i), y = __ldcg(A + (size_t)q * n + i);
                A[(size_t)p * n + i] = c * x - s * y;
                A[(size_t)q * n + i] = s * x + c * y;
            }
            bar.sync();
        }
        if (*(volatile unsigned int*)&rotations[sweep] == 0) break;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *sweeps_done = sweep;
}

// sigma_j = |g_j| (f64 accumulation)
template <typename T>
__global__ void __launch_bounds__(128) column_norms_kernel(const T* __restrict__ Gt, int m, int n, double* __restrict__ norms) {
    const int j = blockIdx.x;
    double a = 0, b = 0, c = 0;
    for (int i = threadIdx.x; i < m; i += 128) {
        const double x = (double)Gt[(size_t)j * m + i];
        a += x * x;
    }
    block_sum3<128>(a, b, c);
    if (threadIdx.x == 0) norms[j] = sqrt(a);
}

// out (rows x ncols, row-major) column j = src row perm[j] (length rows) scaled by scale[perm[j]] (or 1)
template <typename T>
__global__ void __launch_bounds__(256) gather_columns_kernel(const T* __restrict__ src_t, int rows, int ncols, const int* __restrict__ perm,
                                                             const double* __restrict__ inv_scale, T* __restrict__ out, int out_cols) {
    const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
    if (t >= (long long)rows * ncols) return;
    const int i = (int)(t / ncols), j = (int)(t - (long long)i * ncols);
    const int sj = perm[j];
    const double v = (double)src_t[(size_t)sj * rows + i] * (inv_scale ? inv_scale[sj] : 1.0);
    out[(size_t)i * out_cols + j] = (T)v;
}

template <typename T>
__global__ void __launch_bounds__(256) transpose_kernel(const T* __restrict__ a, int rows, int cols, T* __restrict__ at) {
    const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
    if (t >= (long long)rows * cols) return;
    const int i = (int)(t / cols), j = (int)(t - (long long)i * cols);
    at[(size_t)j * rows + i] = a[t];
}

template <typename T>
__global__ void __launch_bounds__(256) identity_kernel(T* __restrict__ v, int n) {
    const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
    if (t >= (long long)n * n) return;
    v[t] = (t / n == t % n) ? (T)1 : (T)0;
}

// Two columns stored in T count as orthogonal when |a_p . a_q| <= sqrt(m) eps |a_p| |a_q|: that is the size of the rounding noise
// their m stored products carry (the criterion of LAPACK's xGESVJ); asking for less only rotates noise until the sweep limit.
template <typename T>
double jacobi_tol(int m) {
    return std::sqrt((double)(m > 1 ? m : 1)) * (double)std::numeric_limits<T>::epsilon();
}

// ---- host twins of the same algorithm (tiny matrices) --------------------------------------------------------------
template <typename T>
int svd_jacobi_host(std::vector<T>& Gt, std::vector<T>& Vt, int m, int n, bool with_v, double abs_floor) {
    const int np = n + (n & 1);
    const double tol = jacobi_tol<T>(m);
    int sweep = 0;
    for (; sweep < kMaxSweeps; ++sweep) {
        unsigned rot = 0;
        for (int r = 0; r < np - 1; ++r)
            for (int k = 0; k < np / 2; ++k) {
                int p, q;
                tournament_pair(np, r, k, p, q);
                if (q >= n) continue;
                T* gp = &Gt[(size_t)p * m];
                T* gq = &Gt[(size_t)q * m];
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < m; ++i) { const double x = gp[i], y = gq[i]; alpha += x * x; beta += y * y; gamma += x * y; }
                T c, s;
                if (!hestenes_rotation<T>(alpha, beta, gamma, tol, abs_floor, c, s)) continue;
                ++rot;
                for (int i = 0; i < m; ++i) { const T x = gp[i], y = gq[i]; gp[i] = c * x - s * y; gq[i] = s * x + c * y; }
                if (with_v) {
                    T* vp = &Vt[(size_t)p * n];
                    T* vq = &Vt[(size_t)q * n];
                    for (int i = 0; i < n; ++i) { const T x = vp[i], y = vq[i]; vp[i] = c * x - s * y; vq[i] = s * x + c * y; }
                }
            }
        if (rot == 0) break;
    }
    return sweep;
}

template <typename T>
int eigh_jacobi_host(std::vector<T>& A, std::vector<T>& Vt, int n, double tiny) {
    const int np = n + (n & 1);
    int sweep = 0;
    for (; sweep < kMaxSweeps; ++sweep) {
        unsigned rot = 0;
        for (int r = 0; r < np - 1; ++r)
            for (int k = 0; k < np / 2; ++k) {
                int p, q;
                tournament_pair(np, r, k, p, q);
                if (q >= n) continue;
                T c, s;
                if (!symmetric_rotation<T>((double)A[(size_t)p * n + p], (double)A[(size_t)q * n + q], (double)A[(size_t)p * n + q], tiny, c, s)) continue;
                ++rot;
                for (int i = 0; i < n; ++i) {
                    const T x = A[(size_t)i * n + p], y = A[(size_t)i * n + q];
                    A[(size_t)i * n + p] = c * x - s * y;
                    A[(size_t)i * n + q] = s * x + c * y;
                    const T vx = Vt[(size_t)p * n + i], vy = Vt[(size_t)q * n + i];
                    Vt[(size_t)p * n + i] = c * vx - s * vy;
                    Vt[(size_t)q * n + i] = s * vx + c * vy;
                }
                for (int i = 0; i < n; ++i) {
                    const T x = A[(size_t)p * n + i], y = A[(size_t)q * n + i];
                    A[(size_t)p * n + i] = c * x - s * y;
                    A[(size_t)q * n + i] = s * x + c * y;
                }
            }
        if (rot == 0) break;
    }
    return sweep;
}

// ---- drivers -------------------------------------------------------------------------------------------------------
struct JacobiWork {   // device scratch shared by the two drivers, stream-ordered on the caller's stream
    Scratch mem;
    unsigned int* sync = nullptr;   // [0] barrier counter, [1 .. kMaxSweeps] rotations per sweep, then sweeps_done
    int init(cudaStream_t s) {
        int rc = mem.alloc((kMaxSweeps + 4) * sizeof(unsigned int), s);
        if (rc) return rc;
        sync = mem.as<unsigned int>();
        return ZB_OK;
    }
    int reset(cudaStream_t s) {
        ZB_CUDA(cudaMemsetAsync(sync, 0, (kMaxSweeps + 4) * sizeof(unsigned int), s));
        return ZB_OK;
    }
    unsigned int* barrier() { return sync; }
    unsigned int* rotations() { return sync + 1; }
    int* sweeps() { return reinterpret_cast<int*>(sync + 1 + kMaxSweeps); }
};

template <typename K>
int cooperative_grid(K kernel, int threads, int wanted, int* grid) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    int per_sm = 0;
    ZB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0));
    const int cap = per_sm * di.sm_count;
    if (cap < 1) return ZB_ERR_DEVICE_FAILURE;
    *grid = std::max(1, std::min(wanted, cap));   // the in-kernel barrier needs every CTA resident: cooperative launch enforces it
    return ZB_OK;
}

// Factorises the m x n (m >= n) matrix whose TRANSPOSE is in dGt (n rows of length m, overwritten).  On return dGt holds the
// rotated columns, dVt (n x n, rows = columns of V) the right vectors when with_v; *sweeps >= kMaxSweeps means no convergence.
template <typename T>
int svd_jacobi_device(T* dGt, T* dVt, int m, int n, bool with_v, double abs_floor, int* sweeps, cudaStream_t s) {
    constexpr int NT = 128;
    JacobiWork w;
    int rc = w.init(s);
    if (rc) return rc;
    if ((rc = w.reset(s))) return rc;
    if (with_v) {
        identity_kernel<T><<<div_up((size_t)n * n, 256), 256, 0, s>>>(dVt, n);
        ZB_LAUNCHED();
    }
    if (g_tune_jacobi_cluster.load()) {   // the whole problem in the shared memory of one 8-CTA cluster?
        const int np = n + (n & 1), cpc = (np + kClusterCtas - 1) / kClusterCtas;
        const size_t smem = (size_t)cpc * ((size_t)m + (with_v ? (size_t)n : 0)) * sizeof(T) + 16;
        if (n >= 32 && smem <= 200 * 1024) {
            auto kern = jacobi_svd_cluster_kernel<T>;
            if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess) {
                cudaLaunchConfig_t cfg = {};
                cfg.gridDim = dim3(kClusterCtas);
                cfg.blockDim = dim3(kClusterThreads);
                cfg.dynamicSmemBytes = smem;
                cfg.stream = s;
                cudaLaunchAttribute attr[1];
                attr[0].id = cudaLaunchAttributeClusterDimension;
                attr[0].val.clusterDim.x = kClusterCtas;
                attr[0].val.clusterDim.y = 1;
                attr[0].val.clusterDim.z = 1;
                cfg.attrs = attr;
                cfg.numAttrs = 1;
                int wv = with_v ? 1 : 0;
                double tol = jacobi_tol<T>(m);
                unsigned int* rots = w.rotations();
                int* sw = w.sweeps();
                if (cudaLaunchKernelEx(&cfg, kern, dGt, dVt, m, n, wv, tol, abs_floor, rots, sw) == cudaSuccess) {
                    ZB_LAUNCHED();
                    ZB_CUDA(cudaMemcpyAsync(sweeps, sw, sizeof(int), cudaMemcpyDeviceToHost, s));
                    ZB_CUDA(cudaStreamSynchronize(s));
                    t_last_kernel = "jacobi_svd_cluster";
                    return ZB_OK;
                }
                (void)cudaGetLastError();   // no cluster of that size on this device: the cooperative kernels below
            }
        }
    }
    int grid = 1;
    const bool warp_pairs = m <= 2048;   // short columns: a warp per pair, four pairs per CTA
    const int pairs = (n + 1) / 2;
    if (warp_pairs) rc = cooperative_grid(jacobi_svd_warp_kernel<T, NT>, NT, (pairs + NT / 32 - 1) / (NT / 32), &grid);
    else rc = cooperative_grid(jacobi_svd_kernel<T, NT>, NT, pairs, &grid);
    if (rc) return rc;
    int wv = with_v ? 1 : 0;
    double tol = jacobi_tol<T>(m);
    unsigned int* bc = w.barrier();
    unsigned int* rots = w.rotations();
    int* sw = w.sweeps();
    void* args[] = {&dGt, &dVt, &m, &n, &wv, &tol, &abs_floor, &bc, &rots, &sw};
    ZB_CUDA(cudaLaunchCooperativeKernel(warp_pairs ? (void*)jacobi_svd_warp_kernel<T, NT> : (void*)jacobi_svd_kernel<T, NT>, dim3(grid), dim3(NT), args, 0, s));
    ZB_LAUNCHED();
    ZB_CUDA(cudaMemcpyAsync(sweeps, sw, sizeof(int), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    t_last_kernel = "jacobi_svd_onesided";
    return ZB_OK;
}

// Completes `have` orthonormal columns of U (m x ucols row-major, f64 work copy) to `ucols` columns: Gram-Schmidt of unit vectors.
void complete_basis(std::vector<double>& u, int m, int ucols, std::vector<char>& valid) {
    int next_e = 0;
    for (int j = 0; j < ucols; ++j) {
        if (valid[j]) continue;
        for (; next_e < m; ++next_e) {
            std::vector<double> v(m, 0.0);
            v[next_e] = 1.0;
            for (int pass = 0; pass < 2; ++pass)   // twice is enough
                for (int k = 0; k < ucols; ++k) {
                    if (!valid[k]) continue;
                    double d = 0;
                    for (int i = 0; i < m; ++i) d += v[i] * u[(size_t)i * ucols + k];
                    for (int i = 0; i < m; ++i) v[i] -= d * u[(size_t)i * ucols + k];
                }
            double nrm = 0;
            for (int i = 0; i < m; ++i) nrm += v[i] * v[i];
            nrm = std::sqrt(nrm);
            if (nrm > 1e-3) {
                for (int i = 0; i < m; ++i) u[(size_t)i * ucols + j] = v[i] / nrm;
                valid[j] = 1;
                ++next_e;
                break;
            }
        }
    }
}

// Host-pointer SVD.  a: m x n row-major.  u: m x ucols; s: n; v: n x n.
template <typename T>
int svd_entry(const T* a, uint32_t m, uint32_t n, int mode, int with_v, T* u, T* s, T* v, uint64_t* converged) {
    if (!a || !s) return ZB_ERR_INVALID_ARGUMENT;
    if (m < n) return ZB_ERR_DIMENSION_MISMATCH;  // svd.zig:86
    if (mode < ZB_SVD_NO_U || mode > ZB_SVD_FULL_U) return ZB_ERR_INVALID_ARGUMENT;
    if (mode != ZB_SVD_NO_U && !u) return ZB_ERR_INVALID_ARGUMENT;
    if (with_v && !v) return ZB_ERR_INVALID_ARGUMENT;
    if (converged) *converged = 0;
    if (n == 0) return ZB_OK;
    const bool want_u = mode != ZB_SVD_NO_U;
    const uint32_t ucols = mode == ZB_SVD_FULL_U ? m : n;
    std::vector<T> Gt((size_t)n * m), Vt(with_v ? (size_t)n * n : 1, (T)0);
    for (uint32_t i = 0; i < m; ++i)
        for (uint32_t j = 0; j < n; ++j) Gt[(size_t)j * m + i] = a[(size_t)i * n + j];
    double frob2 = 0;
    for (const T x : Gt) frob2 += (double)x * (double)x;
    const double eps_t = (double)std::numeric_limits<T>::epsilon();
    const double abs_floor = (double)n * eps_t * eps_t * frob2;
    int sweeps = 0;
    if (n < kDeviceMinN) {
        if (with_v) for (uint32_t j = 0; j < n; ++j) Vt[(size_t)j * n + j] = 1;
        sweeps = svd_jacobi_host<T>(Gt, Vt, (int)m, (int)n, with_v != 0, abs_floor);
    } else {
        DeviceInfo di;
        int rc = device_info(&di);
        if (rc) return rc;
        cudaStream_t st = nullptr;   // default stream: this entry point is synchronous
        Scratch dg, dv;
        if ((rc = dg.alloc(Gt.size() * sizeof(T), st))) return rc;
        if ((rc = dv.alloc(Vt.size() * sizeof(T), st))) return rc;
        ZB_CUDA(cudaMemcpyAsync(dg.p, Gt.data(), Gt.size() * sizeof(T), cudaMemcpyHostToDevice, st));
        if ((rc = svd_jacobi_device<T>(dg.as<T>(), dv.as<T>(), (int)m, (int)n, with_v != 0, abs_floor, &sweeps, st))) return rc;
        ZB_CUDA(cudaMemcpyAsync(Gt.data(), dg.p, Gt.size() * sizeof(T), cudaMemcpyDeviceToHost, st));
        if (with_v) ZB_CUDA(cudaMemcpyAsync(Vt.data(), dv.p, Vt.size() * sizeof(T), cudaMemcpyDeviceToHost, st));
        ZB_CUDA(cudaStreamSynchronize(st));
    }
    t_last_sweeps = sweeps;
    if (sweeps >= kMaxSweeps && converged) *converged = 1;   // svd.zig:79: index of the value that failed (any non-zero = failure)
    // singular values, descending order (svd.zig:463-496)
    std::vector<double> sig(n);
    for (uint32_t j = 0; j < n; ++j) {
        double acc = 0;
        for (uint32_t i = 0; i < m; ++i) { const double x = Gt[(size_t)j * m + i]; acc += x * x; }
        sig[j] = std::sqrt(acc);
    }
    std::vector<int> perm(n);
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(), [&](int x, int y) { return sig[x] > sig[y]; });
    for (uint32_t j = 0; j < n; ++j) s[j] = (T)sig[perm[j]];
    if (with_v)
        for (uint32_t i = 0; i < n; ++i)
            for (uint32_t j = 0; j < n; ++j) v[(size_t)i * n + j] = Vt[(size_t)perm[j] * n + i];
    if (want_u) {
        std::vector<double> uw((size_t)m * ucols, 0.0);
        std::vector<char> valid(ucols, 0);
        const double floor_ = sig[perm[0]] * (double)std::numeric_limits<T>::epsilon() * (double)m;
        for (uint32_t j = 0; j < n; ++j) {
            const int sj = perm[j];
            if (sig[sj] > floor_ && sig[sj] > 0) {
                for (uint32_t i = 0; i < m; ++i) uw[(size_t)i * ucols + j] = (double)Gt[(size_t)sj * m + i] / sig[sj];
                valid[j] = 1;
            }
        }
        complete_basis(uw, (int)m, (int)ucols, valid);   // null-space columns and the m - n extra columns of the full U
        for (size_t i = 0; i < uw.size(); ++i) u[i] = (T)uw[i];
    }
    return ZB_OK;
}

// Device-pointer SVD of a square or tall matrix already on the device (PCA: the covariance never leaves the GPU).
// d_a: m x n row-major (not modified); d_u: m x n (skinny) or null; d_s: n; d_v: n x n or null.  Waits for the stream.
template <typename T>
int svd_device_entry(const T* d_a, uint32_t m, uint32_t n, T* d_u, T* d_s, T* d_v, uint64_t* converged, cudaStream_t st) {
    if (!d_a || !d_s) return ZB_ERR_INVALID_ARGUMENT;
    if (m < n) return ZB_ERR_DIMENSION_MISMATCH;
    if (converged) *converged = 0;
    if (n == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    Scratch dg, dv, dn, dp, dinv;
    if ((rc = dg.alloc((size_t)n * m * sizeof(T), st))) return rc;
    if ((rc = dv.alloc((size_t)n * n * sizeof(T), st))) return rc;
    if ((rc = dn.alloc((size_t)n * sizeof(double), st))) return rc;
    if ((rc = dp.alloc((size_t)n * sizeof(int), st))) return rc;
    if ((rc = dinv.alloc((size_t)n * sizeof(double), st))) return rc;
    transpose_kernel<T><<<div_up((size_t)m * n, 256), 256, 0, st>>>(d_a, (int)m, (int)n, dg.as<T>());
    ZB_LAUNCHED();
    // |A|_F from the column norms (one small read-back) for the noise floor of rank-deficient inputs
    column_norms_kernel<T><<<n, 128, 0, st>>>(dg.as<T>(), (int)m, (int)n, dn.as<double>());
    ZB_LAUNCHED();
    std::vector<double> sig(n), inv(n);
    ZB_CUDA(cudaMemcpyAsync(sig.data(), dn.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    ZB_CUDA(cudaStreamSynchronize(st));
    double frob2 = 0;
    for (double x : sig) frob2 += x * x;
    const double eps_t = (double)std::numeric_limits<T>::epsilon();
    int sweeps = 0;
    if ((rc = svd_jacobi_device<T>(dg.as<T>(), dv.as<T>(), (int)m, (int)n, d_v != nullptr, (double)n * eps_t * eps_t * frob2, &sweeps, st))) return rc;
    t_last_sweeps = sweeps;
    if (sweeps >= kMaxSweeps && converged) *converged = 1;
    column_norms_kernel<T><<<n, 128, 0, st>>>(dg.as<T>(), (int)m, (int)n, dn.as<double>());
    ZB_LAUNCHED();
    ZB_CUDA(cudaMemcpyAsync(sig.data(), dn.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    ZB_CUDA(cudaStreamSynchronize(st));
    std::vector<int> perm(n);
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(), [&](int x, int y) { return sig[x] > sig[y]; });
    // the host entry's noise floor: a column at or below it is rounding noise of a rank-deficient matrix, not a direction of U
    const double floor_ = sig[perm[0]] * eps_t * (double)m;
    bool deficient = false;
    std::vector<T> sorted(n);
    for (uint32_t j = 0; j < n; ++j) {
        sorted[j] = (T)sig[perm[j]];
        const bool keep = sig[j] > floor_ && sig[j] > 0;
        inv[j] = keep ? 1.0 / sig[j] : 0.0;
        deficient |= !keep;
    }
    ZB_CUDA(cudaMemcpyAsync(d_s, sorted.data(), n * sizeof(T), cudaMemcpyHostToDevice, st));
    ZB_CUDA(cudaMemcpyAsync(dp.p, perm.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    ZB_CUDA(cudaMemcpyAsync(dinv.p, inv.data(), n * sizeof(double), cudaMemcpyHostToDevice, st));
    std::vector<T> ut;
    if (d_u) {
        gather_columns_kernel<T><<<div_up((size_t)m * n, 256), 256, 0, st>>>(dg.as<T>(), (int)m, (int)n, dp.as<int>(), dinv.as<double>(), d_u, (int)n);
        ZB_LAUNCHED();
        if (deficient) {   // rare: the null-space columns (zero above) are completed to an orthonormal basis on the host, as svd_entry does
            ut.resize((size_t)m * n);
            ZB_CUDA(cudaMemcpyAsync(ut.data(), d_u, ut.size() * sizeof(T), cudaMemcpyDeviceToHost, st));
            ZB_CUDA(cudaStreamSynchronize(st));
            std::vector<double> uw(ut.begin(), ut.end());
            std::vector<char> valid(n);
            for (uint32_t j = 0; j < n; ++j) valid[j] = inv[perm[j]] != 0.0;
            complete_basis(uw, (int)m, (int)n, valid);
            for (size_t i = 0; i < uw.size(); ++i) ut[i] = (T)uw[i];
            ZB_CUDA(cudaMemcpyAsync(d_u, ut.data(), ut.size() * sizeof(T), cudaMemcpyHostToDevice, st));
        }
    }
    if (d_v) {
        gather_columns_kernel<T><<<div_up((size_t)n * n, 256), 256, 0, st>>>(dv.as<T>(), (int)n, (int)n, dp.as<int>(), nullptr, d_v, (int)n);
        ZB_LAUNCHED();
    }
    ZB_CUDA(cudaStreamSynchronize(st));   // the host vectors above are pageable sources
    return ZB_OK;
}

// Matrix.eigh: validation as the reference orders it (eigen.zig:36-54), then the parallel two-sided Jacobi.
template <typename T>
int eigh_entry(const T* a, uint32_t rows, uint32_t cols, T* values, T* vectors) {
    if (!values || !vectors || (!a && rows)) return ZB_ERR_INVALID_ARGUMENT;
    if (rows != cols) return ZB_ERR_NOT_SQUARE;                                    // :36
    const uint32_t n = rows;
    if (n == 0) return ZB_OK;
    const size_t nn = (size_t)n * n;
    const T eps = std::numeric_limits<T>::epsilon();
    T max_abs = 0;
    for (size_t i = 0; i < nn; ++i) {                                              // :45-50
        if (!std::isfinite(a[i])) return ZB_ERR_NOT_FINITE;
        max_abs = std::max(max_abs, std::fabs(a[i]));
    }
    const T sym_tol = max_abs * std::sqrt(eps);                                    // :51-54
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = i + 1; j < n; ++j)
            if (std::fabs(a[(size_t)i * n + j] - a[(size_t)j * n + i]) > sym_tol) return ZB_ERR_NOT_SYMMETRIC;
    // work on the symmetrised matrix; an off-diagonal entry below eps^2-scale of the Frobenius norm no longer moves an eigenvalue
    std::vector<T> A(nn), Vt(nn, (T)0);
    double frob = 0;
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = 0; j < n; ++j) {
            const T x = (T)(((double)a[(size_t)i * n + j] + (double)a[(size_t)j * n + i]) * 0.5);
            A[(size_t)i * n + j] = x;
            frob += (double)x * (double)x;
        }
    // the reference stops when the off-diagonal Frobenius norm^2 <= |A|_F^2 eps^2 (eigen.zig:64-72); an entry below eps |A|_F / n can
    // no longer lift it above that, and rotating it would only feed rounding noise back in
    const double tiny = std::sqrt(frob) * (double)eps / (double)n;
    for (uint32_t i = 0; i < n; ++i) Vt[(size_t)i * n + i] = 1;
    if (n < kDeviceMinN) {
        t_last_sweeps = eigh_jacobi_host<T>(A, Vt, (int)n, tiny);
    } else {
        constexpr int NT = 128;
        DeviceInfo di;
        int rc = device_info(&di);
        if (rc) return rc;
        cudaStream_t st = nullptr;
        Scratch da, dv, dcs;
        if ((rc = da.alloc(nn * sizeof(T), st))) return rc;
        if ((rc = dv.alloc(nn * sizeof(T), st))) return rc;
        if ((rc = dcs.alloc((size_t)(n + 1) * sizeof(T), st))) return rc;
        JacobiWork w;
        if ((rc = w.init(st))) return rc;
        if ((rc = w.reset(st))) return rc;
        ZB_CUDA(cudaMemcpyAsync(da.p, A.data(), nn * sizeof(T), cudaMemcpyHostToDevice, st));
        ZB_CUDA(cudaMemcpyAsync(dv.p, Vt.data(), nn * sizeof(T), cudaMemcpyHostToDevice, st));
        int grid = 1;
        const int wanted = (int)std::min<size_t>((nn / 2 + NT - 1) / NT, 4096);
        if ((rc = cooperative_grid(jacobi_eigh_kernel<T, NT>, NT, wanted, &grid))) return rc;
        T* pa = da.as<T>();
        T* pv = dv.as<T>();
        T* pcs = dcs.as<T>();
        int ni = (int)n;
        double tn = tiny;
        unsigned int* bc = w.barrier();
        unsigned int* rots = w.rotations();
        int* sw = w.sweeps();
        void* args[] = {&pa, &pv, &ni, &tn, &pcs, &bc, &rots, &sw};
        ZB_CUDA(cudaLaunchCooperativeKernel((void*)jacobi_eigh_kernel<T, NT>, dim3(grid), dim3(NT), args, 0, st));
        ZB_LAUNCHED();
        ZB_CUDA(cudaMemcpyAsync(A.data(), da.p, nn * sizeof(T), cudaMemcpyDeviceToHost, st));
        ZB_CUDA(cudaMemcpyAsync(Vt.data(), dv.p, nn * sizeof(T), cudaMemcpyDeviceToHost, st));
        ZB_CUDA(cudaMemcpyAsync(&t_last_sweeps, sw, sizeof(int), cudaMemcpyDeviceToHost, st));
        ZB_CUDA(cudaStreamSynchronize(st));
        t_last_kernel = "jacobi_eigh_twosided";
    }
    // ascending eigenvalues, matching eigenvectors as columns (eigen.zig:114-133)
    std::vector<int> perm(n);
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(), [&](int x, int y) { return A[(size_t)x * n + x] < A[(size_t)y * n + y]; });
    for (uint32_t j = 0; j < n; ++j) {
        values[j] = A[(size_t)perm[j] * n + perm[j]];
        for (uint32_t i = 0; i < n; ++i) vectors[(size_t)i * n + j] = Vt[(size_t)perm[j] * n + i];
    }
    return ZB_OK;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" {

int zb_last_sweeps(void) { return t_last_sweeps; }

int zb_svd_f64(const double* a, uint32_t m, uint32_t n, int mode, int with_v, double* u, double* s, double* v, uint64_t* converged) {
    return svd_entry<double>(a, m, n, mode, with_v, u, s, v, converged);
}
int zb_svd_f32(const float* a, uint32_t m, uint32_t n, int mode, int with_v, float* u, float* s, float* v, uint64_t* converged) {
    return svd_entry<float>(a, m, n, mode, with_v, u, s, v, converged);
}
int zb_svd_dev_f64(const double* d_a, uint32_t m, uint32_t n, double* d_u, double* d_s, double* d_v, uint64_t* converged, zb_stream s) {
    return svd_device_entry<double>(d_a, m, n, d_u, d_s, d_v, converged, (cudaStream_t)s);
}
int zb_svd_dev_f32(const float* d_a, uint32_t m, uint32_t n, float* d_u, float* d_s, float* d_v, uint64_t* converged, zb_stream s) {
    return svd_device_entry<float>(d_a, m, n, d_u, d_s, d_v, converged, (cudaStream_t)s);
}
int zb_eigh_f64(const double* a, uint32_t rows, uint32_t cols, double* values, double* vectors) {
    return eigh_entry<double>(a, rows, cols, values, vectors);
}
int zb_eigh_f32(const float* a, uint32_t rows, uint32_t cols, float* values, float* vectors) {
    return eigh_entry<float>(a, rows, cols, values, vectors);
}

}  // extern "C"
