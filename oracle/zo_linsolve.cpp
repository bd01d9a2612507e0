// zo_linsolve.cpp -- CPU oracle of Matrix.lu, LuResult.solve, det, inv and chol (reference src/matrix/Matrix.zig:67-85, 376-441,
// 511-583, 1156-1365), restated with the reference's loops, comparisons and operation order.  Built with -ffp-contract=off (Makefile):
// the reference never fuses a multiply and an add.  Matrices are row-major n x n (b and x: n x k).  Returns 0, or the library's status
// codes 32 (Singular) and 33 (NotPositiveDefinite).  TEST INFRASTRUCTURE ONLY.
#include <cmath>
#include <cstdint>
#include <limits>
#include <utility>
#include <vector>

namespace {

constexpr int kSingular = 32, kNotPositiveDefinite = 33;

template <typename T> constexpr T eps() { return std::numeric_limits<T>::epsilon(); }

// @max(a, b) on floats: a NaN operand yields the other operand
template <typename T> T zmax(T a, T b) { return std::isnan(a) ? b : std::isnan(b) ? a : (a > b ? a : b); }

// Matrix.lu (:1226-1316): l and u n x n, perm n, *sign
template <typename T>
void lu(const T* a, int n, T* l, T* u, uint32_t* perm, T* sign) {
    std::vector<T> work(a, a + (size_t)n * n);
    auto W = [&](int i, int j) -> T& { return work[(size_t)i * n + j]; };
    for (size_t e = 0; e < (size_t)n * n; ++e) l[e] = u[e] = 0;
    for (int i = 0; i < n; ++i) { l[(size_t)i * n + i] = 1; perm[i] = (uint32_t)i; }
    T s = 1;
    for (int k = 0; k < n; ++k) {
        int max_row = k;
        T max_val = std::fabs(W(k, k));
        for (int r = k + 1; r < n; ++r) {
            const T v = std::fabs(W(r, k));
            if (v > max_val) { max_val = v; max_row = r; }
        }
        if (max_row != k) {
            s = -s;
            std::swap(perm[k], perm[max_row]);
            for (int j = 0; j < n; ++j) std::swap(W(k, j), W(max_row, j));
            for (int j = 0; j < k; ++j) std::swap(l[(size_t)k * n + j], l[(size_t)max_row * n + j]);
        }
        for (int j = k; j < n; ++j) u[(size_t)k * n + j] = W(k, j);
        for (int i = k + 1; i < n; ++i) {
            if (std::fabs(W(k, k)) > eps<T>()) {
                const T factor = W(i, k) / W(k, k);
                l[(size_t)i * n + k] = factor;
                for (int j = k + 1; j < n; ++j) W(i, j) -= factor * W(k, j);
            }
        }
    }
    *sign = s;
}

// LuResult.solve (:1177-1221)
template <typename T>
int lu_solve(const T* l, const T* u, const uint32_t* perm, int n, const T* b, int k, T* x) {
    for (int i = 0; i < n; ++i)
        for (int c = 0; c < k; ++c) x[(size_t)i * k + c] = b[(size_t)perm[i] * k + c];
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < i; ++j) {
            const T lij = l[(size_t)i * n + j];
            for (int c = 0; c < k; ++c) x[(size_t)i * k + c] -= lij * x[(size_t)j * k + c];
        }
    T u_max = 0;
    for (int r = 0; r < n; ++r)
        for (int c = r; c < n; ++c) u_max = zmax(u_max, (T)std::fabs(u[(size_t)r * n + c]));
    if (u_max == 0) return kSingular;
    const T tol = u_max * eps<T>() * 100;
    for (int i = n - 1; i >= 0; --i) {
        const T pivot = u[(size_t)i * n + i];
        if (std::fabs(pivot) < tol) return kSingular;
        for (int j = i + 1; j < n; ++j) {
            const T uij = u[(size_t)i * n + j];
            for (int c = 0; c < k; ++c) x[(size_t)i * k + c] -= uij * x[(size_t)j * k + c];
        }
        for (int c = 0; c < k; ++c) x[(size_t)i * k + c] /= pivot;
    }
    return 0;
}

// Matrix.det (:1336-1365), n >= 1
template <typename T>
T det(const T* a, int n) {
    auto m = [&](int i, int j) { return a[(size_t)i * n + j]; };
    if (n == 1) return m(0, 0);
    if (n == 2) return m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0);
    if (n == 3)
        return m(0, 0) * m(1, 1) * m(2, 2) + m(0, 1) * m(1, 2) * m(2, 0) + m(0, 2) * m(1, 0) * m(2, 1) - m(0, 2) * m(1, 1) * m(2, 0) -
               m(0, 1) * m(1, 0) * m(2, 2) - m(0, 0) * m(1, 2) * m(2, 1);
    std::vector<T> l((size_t)n * n), u((size_t)n * n);
    std::vector<uint32_t> p(n);
    T d;
    lu(a, n, l.data(), u.data(), p.data(), &d);
    for (int i = 0; i < n; ++i) d *= u[(size_t)i * n + i];
    return d;
}

// Matrix.inv (:376-427) and inverseGaussJordan (:513-583), n >= 1
template <typename T>
int inv(const T* a, int n, T* out) {
    auto m = [&](int i, int j) { return a[(size_t)i * n + j]; };
    const T e = eps<T>();
    if (n == 1) {
        const T d = m(0, 0);
        if (std::fabs(d) < e) return kSingular;
        out[0] = 1 / d;
        return 0;
    }
    if (n == 2) {
        const T d = m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0);
        if (std::fabs(d) < e) return kSingular;
        out[0] = m(1, 1) / d; out[1] = -m(0, 1) / d; out[2] = -m(1, 0) / d; out[3] = m(0, 0) / d;
        return 0;
    }
    if (n == 3) {
        const T c00 = m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1);
        const T c01 = m(0, 2) * m(2, 1) - m(0, 1) * m(2, 2);
        const T c02 = m(0, 1) * m(1, 2) - m(0, 2) * m(1, 1);
        const T d = m(0, 0) * c00 + m(1, 0) * c01 + m(2, 0) * c02;
        if (std::fabs(d) < e) return kSingular;
        out[0] = c00 / d; out[1] = c01 / d; out[2] = c02 / d;
        out[3] = (m(1, 2) * m(2, 0) - m(1, 0) * m(2, 2)) / d;
        out[4] = (m(0, 0) * m(2, 2) - m(0, 2) * m(2, 0)) / d;
        out[5] = (m(0, 2) * m(1, 0) - m(0, 0) * m(1, 2)) / d;
        out[6] = (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0)) / d;
        out[7] = (m(0, 1) * m(2, 0) - m(0, 0) * m(2, 1)) / d;
        out[8] = (m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0)) / d;
        return 0;
    }
    const int w = 2 * n;
    std::vector<T> g((size_t)n * w);
    auto G = [&](int i, int j) -> T& { return g[(size_t)i * w + j]; };
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) { G(i, j) = m(i, j); G(i, n + j) = i == j ? 1 : 0; }
    for (int k = 0; k < n; ++k) {
        int max_row = k;
        T max_val = std::fabs(G(k, k));
        for (int r = k + 1; r < n; ++r) {
            const T v = std::fabs(G(r, k));
            if (v > max_val) { max_val = v; max_row = r; }
        }
        if (max_val < e * 10) return kSingular;
        if (max_row != k)
            for (int j = k; j < w; ++j) std::swap(G(k, j), G(max_row, j));
        const T pivot = G(k, k);
        for (int j = k; j < w; ++j) G(k, j) /= pivot;
        for (int r = 0; r < n; ++r) {
            if (r == k) continue;
            const T factor = G(r, k);
            for (int j = k; j < w; ++j) G(r, j) -= factor * G(k, j);
        }
    }
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) out[(size_t)i * n + j] = G(i, n + j);
    return 0;
}

// Matrix.chol (:1320-1332) over cholesky (:71-85)
template <typename T>
int chol(const T* a, int n, T* l) {
    for (size_t e = 0; e < (size_t)n * n; ++e) l[e] = a[e];
    for (int j = 0; j < n; ++j) {
        T sum = l[(size_t)j * n + j];
        for (int k = 0; k < j; ++k) sum -= l[(size_t)j * n + k] * l[(size_t)j * n + k];
        if (sum <= 0) return kNotPositiveDefinite;
        const T ljj = std::sqrt(sum);
        l[(size_t)j * n + j] = ljj;
        for (int i = j + 1; i < n; ++i) {
            T s = l[(size_t)i * n + j];
            for (int k = 0; k < j; ++k) s -= l[(size_t)i * n + k] * l[(size_t)j * n + k];
            l[(size_t)i * n + j] = s / ljj;
        }
    }
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j) l[(size_t)i * n + j] = 0;
    return 0;
}

}  // namespace

#define ZO_LINSOLVE(T, S)                                                                                                          \
    extern "C" int zo_lu_##S(const T* a, int n, T* l, T* u, uint32_t* perm, T* sign) { lu<T>(a, n, l, u, perm, sign); return 0; }     \
    extern "C" int zo_lu_solve_##S(const T* l, const T* u, const uint32_t* perm, int n, const T* b, int k, T* x) {                   \
        return lu_solve<T>(l, u, perm, n, b, k, x);                                                                                 \
    }                                                                                                                              \
    extern "C" int zo_det_##S(const T* a, int n, T* out) { *out = det<T>(a, n); return 0; }                                        \
    extern "C" int zo_inv_##S(const T* a, int n, T* out) { return inv<T>(a, n, out); }                                             \
    extern "C" int zo_chol_##S(const T* a, int n, T* l) { return chol<T>(a, n, l); }
ZO_LINSOLVE(float, f32)
ZO_LINSOLVE(double, f64)
