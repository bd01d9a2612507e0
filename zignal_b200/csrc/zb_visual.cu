// zb_visual.cu -- Image.diff (image.zig:1139, image/diff.zig:27-203), Image.applyColormap (image.zig:1190-1247, image/colormaps.zig),
// flipLeftRight / flipTopBottom (image/transforms.zig:28-45) and invert (image.zig:494-511, color.zig:328,441) on the device.
//
// All of them are memory-bound passes over row segments.  A block stages one segment of kSegBytes bytes of a row (of each image it
// reads) in shared memory with 16-byte accesses where global and shared addresses agree modulo 16 and byte accesses at the edges,
// works on the pixels there, and writes its output segment back the same way.  So every global access is coalesced whatever the
// pixel size (Rgb(u8) included), and a view is read and written only inside its own pixels.  Row tiles go through row_grid.
//
// diff statistics: kStatBlocks blocks walk the segments, each reduces its samples in a fixed tree order into one partial in
// stream-ordered scratch; one block then merges the partials in block order and the host reads the single result back.  8-bit
// formats accumulate integer sums, so n, sum, min and max are exact and the host rounds mean and variance once from 128-bit
// integers; float formats run Welford per thread and Chan's merge above it, so a repeated call returns the same bits.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

#include <math_constants.h>

#include "zb_convert.cuh"
#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {
namespace {

constexpr int kThreads = 256;
constexpr int kSegBytes = 6144;      // bytes of one staged row segment: a multiple of 16 and of every pixel size (1, 3, 4, 16)
constexpr int kFinalThreads = 512;   // the one block that merges the diff partials
constexpr int kRangeBlocks = 1024;   // blocks of the applyColormap range pass
constexpr int kStatBlocks = 1024;    // blocks of a diff with statistics: fixed, so the merge order (and the result's bits) is too

template <int F> constexpr int pixel_size() { return (int)sizeof(typename Fmt<F>::CT) * Fmt<F>::N; }

// Copies n bytes between global memory g and its shared-memory image sm.  16-byte accesses when sm and g agree modulo 16, byte
// accesses for the unaligned head and tail (and for everything when they do not agree).  Every thread of the block takes part.
template <bool TO_SHARED>
__device__ __forceinline__ void span_copy(uint8_t* sm, uint8_t* g, size_t n) {
    const size_t lead = (16 - ((uintptr_t)g & 15)) & 15, head = lead < n ? lead : n;
    const bool vec = (((uintptr_t)sm ^ (uintptr_t)g) & 15) == 0;
    const size_t nv = vec ? (n - head) / 16 : 0;
    for (size_t i = threadIdx.x; i < head; i += blockDim.x) {
        if (TO_SHARED) sm[i] = g[i]; else g[i] = sm[i];
    }
    uint4* s4 = (uint4*)(sm + head);
    uint4* g4 = (uint4*)(g + head);
    for (size_t v = threadIdx.x; v < nv; v += blockDim.x) {
        if (TO_SHARED) s4[v] = g4[v]; else g4[v] = s4[v];
    }
    for (size_t i = head + nv * 16 + threadIdx.x; i < n; i += blockDim.x) {
        if (TO_SHARED) sm[i] = g[i]; else g[i] = sm[i];
    }
}

// The shared image of a global span: the same address modulo 16 inside a 16-byte aligned buffer.
__device__ __forceinline__ uint8_t* shadow(uint8_t* buf, const void* g) { return buf + ((uintptr_t)g & 15); }

template <int PB>
__device__ __forceinline__ void swap_bytes(uint8_t* x, uint8_t* y) {
#pragma unroll
    for (int k = 0; k < PB; ++k) { const uint8_t t = x[k]; x[k] = y[k]; y[k] = t; }
}

// ---- diff ----------------------------------------------------------------------------------------------------------------------------

struct DiffOpts { float threshold, scale; int binary, force_opaque; };

// Statistics of a set of diff samples.  8-bit formats use cnt / isum / isq / mn / mx; float formats n / mean / m2 / sum / mn / mx.
struct Part {
    unsigned long long n, cnt, isum, isq;
    double mean, m2, sum, mn, mx;
};

__device__ __forceinline__ Part part_identity() {
    Part p;
    p.n = p.cnt = p.isum = p.isq = 0;
    p.mean = p.m2 = p.sum = 0.0;
    p.mn = CUDART_INF;
    p.mx = -CUDART_INF;
    return p;
}

// Chan's pairwise update for (n, mean, m2); the sums add, min / max ignore NaN (Zig's @min / @max, stats.zig:102-103).
__device__ __forceinline__ Part merge(Part a, const Part& b) {
    a.cnt += b.cnt;
    a.isum += b.isum;
    a.isq += b.isq;
    if (b.n) {
        if (!a.n) {
            a.mean = b.mean;
            a.m2 = b.m2;
        } else {
            const double na = (double)a.n, nb = (double)b.n, n = __dadd_rn(na, nb);
            const double delta = __dsub_rn(b.mean, a.mean);
            a.mean = __dadd_rn(a.mean, __dmul_rn(delta, __ddiv_rn(nb, n)));
            a.m2 = __dadd_rn(__dadd_rn(a.m2, b.m2), __dmul_rn(__dmul_rn(delta, delta), __ddiv_rn(__dmul_rn(na, nb), n)));
        }
        a.n += b.n;
        a.sum = __dadd_rn(a.sum, b.sum);
    }
    a.mn = fmin(a.mn, b.mn);
    a.mx = fmax(a.mx, b.mx);
    return a;
}

// One pixel of diff.zig:41-143: writes o (which may alias a or b: every channel is read before any is written) and returns the stats
// sample; *differs is the diff_count test.
template <int F>
__device__ __forceinline__ double diff_pixel(const typename Fmt<F>::CT* a, const typename Fmt<F>::CT* b, typename Fmt<F>::CT* o,
                                             const DiffOpts& op, bool* differs) {
    using CT = typename Fmt<F>::CT;
    constexpr int N = Fmt<F>::N;
    constexpr bool flt = sizeof(CT) == 4;
    const CT max_v = flt ? (CT)1.0f : (CT)255;
    float d[N];
    bool any = false;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        if constexpr (flt) d[k] = fabsf(__fsub_rn((float)a[k], (float)b[k]));                      // @abs(v1 - v2)
        else d[k] = (float)abs((int)a[k] - (int)b[k]);                                             // |v1 - v2| as f32
        any |= d[k] > op.threshold;                                                                // alpha included
    }
    *differs = any;
    if constexpr (N == 1) {                                                                        // :48-79
        CT v;
        if (op.binary) v = any ? max_v : (CT)0;
        else if constexpr (flt) v = __fmul_rn(d[0], op.scale);
        else v = clamp_u8_from_float(__fmul_rn(d[0], op.scale));                                    // meta.clamp
        o[0] = v;
        return (double)v;                                                                          // a NaN f32 enters the stats
    } else {                                                                                       // :80-143
        double pixel_max = 0.0;
#pragma unroll
        for (int k = 0; k < N; ++k) {
            if (N == 4 && k == 3 && op.force_opaque) { o[k] = max_v; continue; }                  // alpha written, not in the max
            CT v;
            if (op.binary) v = any ? max_v : (CT)0;
            else if constexpr (flt) v = __fmul_rn(d[k], op.scale);
            else v = clamp_u8_from_float(__fmul_rn(d[k], op.scale));
            o[k] = v;
            if ((double)v > pixel_max) pixel_max = (double)v;                                      // NaN never enters
        }
        return pixel_max;
    }
}

template <int F, bool STATS>
__global__ void __launch_bounds__(kThreads) diff_kernel(const uint8_t* a, size_t a_pitch, const uint8_t* b,
                                                        size_t b_pitch, uint8_t* o, size_t o_pitch, int rows, int cols, unsigned xblocks,
                                                        DiffOpts op, Part* __restrict__ part) {
    using CT = typename Fmt<F>::CT;
    constexpr int PB = pixel_size<F>(), P = kSegBytes / PB;
    constexpr bool flt = sizeof(CT) == 4;
    __shared__ __align__(16) uint8_t sa[kSegBytes + 16], sb[kSegBytes + 16];
    // Without statistics a block takes the one segment (row tile, blockIdx.x) of a row_grid launch.  With them a fixed number of blocks
    // walk the segments in raster order, so the per-block reduction is paid kStatBlocks times rather than once per segment.
    size_t seg = 0, end = 0, step = 1;
    Part st;
    if (STATS) {
        st = part_identity();
        seg = blockIdx.x;
        end = (size_t)rows * xblocks;
        step = gridDim.x;
    } else {
        const int r = ZB_GRID_ROW();
        if (r >= rows) return;                                                                     // uniform per block
        seg = (size_t)r * xblocks + blockIdx.x;
        end = seg + 1;
    }
    for (; seg < end; seg += step) {
        const size_t r = seg / xblocks;
        const int c0 = (int)(seg - r * xblocks) * P, n = min(P, cols - c0);
        uint8_t* ga = const_cast<uint8_t*>(a) + (size_t)r * a_pitch + (size_t)c0 * PB;
        uint8_t* gb = const_cast<uint8_t*>(b) + (size_t)r * b_pitch + (size_t)c0 * PB;
        uint8_t* go = o + (size_t)r * o_pitch + (size_t)c0 * PB;
        uint8_t *ma = shadow(sa, ga), *mb = shadow(sb, gb);
        span_copy<true>(ma, ga, (size_t)n * PB);
        span_copy<true>(mb, gb, (size_t)n * PB);
        __syncthreads();
        // the output overwrites the staged input whose alignment it shares, so its store can be vectorised
        uint8_t* mo = ((((uintptr_t)go ^ (uintptr_t)ga) & 15) != 0 && (((uintptr_t)go ^ (uintptr_t)gb) & 15) == 0) ? mb : ma;
        for (int j = threadIdx.x; j < n; j += kThreads) {
            bool differs;
            const double x = diff_pixel<F>((const CT*)(ma + j * PB), (const CT*)(mb + j * PB), (CT*)(mo + j * PB), op, &differs);
            if (STATS) {
                st.cnt += differs;
                st.n += 1;
                if constexpr (flt) {                                                                   // Welford, stats.zig:80-105
                    const double delta = __dsub_rn(x, st.mean);
                    st.mean = __dadd_rn(st.mean, __ddiv_rn(delta, (double)st.n));
                    st.m2 = __dadd_rn(st.m2, __dmul_rn(delta, __dsub_rn(x, st.mean)));
                    st.sum = __dadd_rn(st.sum, x);
                } else {
                    const unsigned xi = (unsigned)x;
                    st.isum += xi;
                    st.isq += xi * xi;
                }
                st.mn = fmin(st.mn, x);
                st.mx = fmax(st.mx, x);
            }
        }
        __syncthreads();
        span_copy<false>(mo, go, (size_t)n * PB);
        __syncthreads();                                                                               // before the next segment's loads
    }
    if (STATS) {
        __shared__ Part red[kThreads];
        red[threadIdx.x] = st;
        __syncthreads();
        for (int s = kThreads / 2; s > 0; s >>= 1) {
            if ((int)threadIdx.x < s) red[threadIdx.x] = merge(red[threadIdx.x], red[threadIdx.x + s]);
            __syncthreads();
        }
        if (threadIdx.x == 0) part[blockIdx.x] = red[0];
    }
}

// Merges n partials in block order: thread t folds partials t, t + kFinalThreads, ... in turn, then a fixed tree joins the threads.
__global__ void __launch_bounds__(kFinalThreads) diff_final(const Part* __restrict__ part, size_t n, Part* __restrict__ out) {
    __shared__ Part red[kFinalThreads];
    Part st = part_identity();
    for (size_t i = threadIdx.x; i < n; i += kFinalThreads) st = merge(st, part[i]);
    red[threadIdx.x] = st;
    __syncthreads();
    for (int s = kFinalThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] = merge(red[threadIdx.x], red[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = red[0];
}

// p / q correctly rounded to the nearest double (ties to even); q > 0.
double ratio_to_double(unsigned __int128 p, unsigned __int128 q) {
    if (p == 0) return 0.0;
    unsigned __int128 m = p / q, r = p % q;
    int e = 0;
    bool sticky = false;
    const unsigned __int128 lo = (unsigned __int128)1 << 54, hi = (unsigned __int128)1 << 55;
    while (m >= hi) { sticky |= (m & 1) != 0; m >>= 1; ++e; }
    while (m < lo) {                                                                               // one more quotient bit
        r <<= 1;
        m <<= 1;
        if (r >= q) { r -= q; m |= 1; }
        --e;
    }
    sticky |= r != 0;
    // m holds 55 significant bits: 53 kept, a guard bit and a round bit
    uint64_t keep = (uint64_t)(m >> 2);
    const unsigned low = (unsigned)(m & 3);
    if (low > 2 || (low == 2 && (sticky || (keep & 1)))) ++keep;
    return std::ldexp((double)keep, e + 2);
}

template <int F>
int run_diff(const zb_image* a, const zb_image* b, zb_image* out, const DiffOpts& op, zb_diff_stats* stats, cudaStream_t s) {
    constexpr int PB = pixel_size<F>(), P = kSegBytes / PB;
    constexpr bool flt = F == ZB_PIX_F32 || F == ZB_PIX_RGBAF32;
    const size_t rows = a->rows, cols = a->cols, n = rows * cols;
    if (n == 0) {
        if (stats) memset(stats, 0, sizeof(*stats));
        return ZB_OK;
    }
    const unsigned xblocks = div_up(cols, P);
    const size_t blocks = std::min<size_t>(kStatBlocks, (size_t)xblocks * rows);
    const uint8_t *pa = (const uint8_t*)a->data, *pb = (const uint8_t*)b->data;
    uint8_t* po = (uint8_t*)out->data;
    if (!stats) {
        diff_kernel<F, false><<<row_grid(xblocks, rows), kThreads, 0, s>>>(pa, a->stride * PB, pb, b->stride * PB, po, out->stride * PB,
                                                                           (int)rows, (int)cols, xblocks, op, nullptr);
        ZB_LAUNCHED();
        t_last_kernel = "diff";
        return ZB_OK;
    }
    DeviceInfo di;                                                                                 // keeps the pool's memory between calls
    int rc = device_info(&di);
    if (rc) return rc;
    Scratch buf;
    if ((rc = buf.alloc((blocks + 1) * sizeof(Part), s))) return rc;
    Part* part = buf.as<Part>();
    diff_kernel<F, true><<<(unsigned)blocks, kThreads, 0, s>>>(pa, a->stride * PB, pb, b->stride * PB, po, out->stride * PB, (int)rows,
                                                               (int)cols, xblocks, op, part);
    ZB_LAUNCHED();
    diff_final<<<1, kFinalThreads, 0, s>>>(part, blocks, part + blocks);
    ZB_LAUNCHED();
    Part h;
    ZB_CUDA(cudaMemcpyAsync(&h, part + blocks, sizeof(Part), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    stats->n = n;
    stats->diff_count = h.cnt;
    stats->min = h.mn;                                                                             // n > 0 here (stats.zig:167-178)
    stats->max = h.mx;
    if (flt) {
        stats->sum = h.sum;
        stats->mean = h.mean;
        stats->variance = n > 1 ? h.m2 / (double)(n - 1) : 0.0;
    } else {
        // exact: mean = S / n, variance = (n Q - S^2) / (n (n - 1)), each rounded once
        const unsigned __int128 S = h.isum, Q = h.isq, N = n;
        stats->sum = (double)h.isum;                                                               // exact below 2^53, as the reference's
        stats->mean = ratio_to_double(S, N);
        stats->variance = n > 1 ? ratio_to_double(N * Q - S * S, N * (N - 1)) : 0.0;
    }
    t_last_kernel = "diff";
    return ZB_OK;
}

// ---- applyColormap ----------------------------------------------------------------------------------------------------------------

struct Lut768 { uint8_t v[768]; };
struct Range { double min, max; };

// The per-pixel key whose order is the order of the reference's scalar: the scalar itself for U8 / F32, the Gray(u8) luma for 8-bit
// colours (scalar = y / 255), the clamped f32 luma for Rgba(f32).  Reuses convertColor's luma sums (zb_convert.cuh).
template <int F>
__device__ __forceinline__ float pixel_key(const typename Fmt<F>::CT* p) {
    if constexpr (F == ZB_PIX_U8 || F == ZB_PIX_F32) return (float)p[0];
    else if constexpr (F == ZB_PIX_RGBAF32) return luma_f32(p[0], p[1], p[2]);
    else return (float)luma_u8(p[0], p[1], p[2]);
}
// meta.as(f64, v) for scalars, convertColor(f64, px) for colours (image.zig:1217,1239; color.zig:133-136 then Gray.as(f64), :548-556)
template <int F>
__device__ __forceinline__ double key_scalar(float key) {
    if constexpr (F == ZB_PIX_RGB8 || F == ZB_PIX_RGBA8) return __ddiv_rn((double)key, 255.0);
    else return (double)key;
}
// meta.normalize (meta.zig:255-260) and the index of colormaps.zig:46-47: round(t * 255).  A NaN quotient (inf / inf) clamps to 1.
__device__ __forceinline__ int colormap_index(double v, double mn, double mx) {
    double t = 0.0;
    if (!(v != v || mn != mn || mx != mx) && !(mx <= mn)) t = clamp01(__ddiv_rn(__dsub_rn(v, mn), __dsub_rn(mx, mn)));
    return (int)round(__dmul_rn(t, 255.0));
}

// Per-block min / max of the keys over the view (NaN ignored).
template <int F>
__global__ void __launch_bounds__(kThreads) colormap_range(const uint8_t* __restrict__ src, size_t pitch, int rows, int cols,
                                                           float2* __restrict__ part) {
    using CT = typename Fmt<F>::CT;
    constexpr int PB = pixel_size<F>();
    float mn = CUDART_INF_F, mx = -CUDART_INF_F;
    for (int r = blockIdx.x; r < rows; r += gridDim.x) {
        const CT* row = (const CT*)(src + (size_t)r * pitch);
        for (int c = threadIdx.x; c < cols; c += kThreads) {
            const float k = pixel_key<F>(row + (size_t)c * (PB / sizeof(CT)));
            mn = fminf(mn, k);
            mx = fmaxf(mx, k);
        }
    }
    __shared__ float2 red[kThreads];
    red[threadIdx.x] = make_float2(mn, mx);
    __syncthreads();
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            red[threadIdx.x].x = fminf(red[threadIdx.x].x, red[threadIdx.x + s].x);
            red[threadIdx.x].y = fmaxf(red[threadIdx.x].y, red[threadIdx.x + s].y);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}

// image.zig:1197-1233: the range, then the table the map kernel gathers from.  8-bit formats get one colour per key (their scalar has
// only 256 values); float formats get the LUT itself and read the range from `range`.
template <int F>
__global__ void __launch_bounds__(kThreads) colormap_setup(const float2* __restrict__ part, int n_part, int has_min, double min_opt,
                                                           int has_max, double max_opt, Lut768 lut, Range* __restrict__ range,
                                                           uint8_t* __restrict__ table) {
    __shared__ float2 red[kThreads];
    __shared__ Range rg;
    float mn = CUDART_INF_F, mx = -CUDART_INF_F;
    for (int i = threadIdx.x; i < n_part; i += kThreads) {
        mn = fminf(mn, part[i].x);
        mx = fmaxf(mx, part[i].y);
    }
    red[threadIdx.x] = make_float2(mn, mx);
    __syncthreads();
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            red[threadIdx.x].x = fminf(red[threadIdx.x].x, red[threadIdx.x + s].x);
            red[threadIdx.x].y = fmaxf(red[threadIdx.x].y, red[threadIdx.x + s].y);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // the scan starts from floatMax / -floatMax (image.zig:1207-1208); an empty partial is +inf / -inf and changes nothing
        const double fmax64 = 1.7976931348623157e308;
        const double min_v = fmin(fmax64, key_scalar<F>(red[0].x)), max_v = fmax(-fmax64, key_scalar<F>(red[0].y));
        double lo = has_min ? min_opt : min_v, hi = has_max ? max_opt : max_v;
        if (hi <= lo) hi = __dadd_rn(lo, 1.0);                                                     // :1231-1233
        rg.min = lo;
        rg.max = hi;
        *range = rg;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 768; k += kThreads) {
        if constexpr (F == ZB_PIX_F32 || F == ZB_PIX_RGBAF32) {
            table[k] = lut.v[k];
        } else {
            const int key = k / 3, ch = k - 3 * key;
            table[k] = lut.v[3 * colormap_index(key_scalar<F>((float)key), rg.min, rg.max) + ch];
        }
    }
}

template <int F>
__global__ void __launch_bounds__(kThreads) colormap_map(const uint8_t* __restrict__ src, size_t pitch, uint8_t* __restrict__ dst,
                                                         size_t dst_pitch, int rows, int cols, const Range* __restrict__ range,
                                                         const uint8_t* __restrict__ table) {
    using CT = typename Fmt<F>::CT;
    constexpr int PB = pixel_size<F>(), P = kSegBytes / PB;
    constexpr bool flt = F == ZB_PIX_F32 || F == ZB_PIX_RGBAF32;
    __shared__ __align__(16) uint8_t si[kSegBytes + 16], so[3 * P + 16];
    __shared__ uint8_t tab[768];
    const int r = ZB_GRID_ROW();
    if (r >= rows) return;
    const int c0 = blockIdx.x * P, n = min(P, cols - c0);
    uint8_t* gi = const_cast<uint8_t*>(src) + (size_t)r * pitch + (size_t)c0 * PB;
    uint8_t* gd = dst + (size_t)r * dst_pitch + (size_t)c0 * 3;
    uint8_t *mi = shadow(si, gi), *md = shadow(so, gd);
    for (int k = threadIdx.x; k < 768; k += kThreads) tab[k] = table[k];
    span_copy<true>(mi, gi, (size_t)n * PB);
    double mn = 0.0, mx = 0.0;
    if (flt) { mn = range->min; mx = range->max; }
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += kThreads) {
        const float key = pixel_key<F>((const CT*)(mi + j * PB));
        const int i = flt ? 3 * colormap_index((double)key, mn, mx) : 3 * (int)key;
        md[3 * j] = tab[i];
        md[3 * j + 1] = tab[i + 1];
        md[3 * j + 2] = tab[i + 2];
    }
    __syncthreads();
    span_copy<false>(md, gd, (size_t)n * 3);
}

template <int F>
int run_colormap(const zb_image* src, const Lut768& lut, int has_min, double min, int has_max, double max, zb_image* dst, cudaStream_t s) {
    constexpr int PB = pixel_size<F>(), P = kSegBytes / PB;
    const int rows = (int)src->rows, cols = (int)src->cols;
    const bool scan = !(has_min && has_max);
    const int n_part = scan ? (int)std::min<size_t>(kRangeBlocks, (size_t)rows) : 0;
    DeviceInfo di;                                                                                 // keeps the pool's memory between calls
    int rc = device_info(&di);
    if (rc) return rc;
    Scratch buf;
    if ((rc = buf.alloc(sizeof(Range) + 768 + (size_t)n_part * sizeof(float2) + 16, s))) return rc;
    Range* range = buf.as<Range>();
    float2* part = (float2*)((uint8_t*)buf.p + sizeof(Range));
    uint8_t* table = (uint8_t*)(part + n_part);
    const uint8_t* ps = (const uint8_t*)src->data;
    if (scan) {
        colormap_range<F><<<n_part, kThreads, 0, s>>>(ps, src->stride * PB, rows, cols, part);
        ZB_LAUNCHED();
    }
    colormap_setup<F><<<1, kThreads, 0, s>>>(part, n_part, has_min, min, has_max, max, lut, range, table);
    ZB_LAUNCHED();
    colormap_map<F><<<row_grid(div_up(cols, P), rows), kThreads, 0, s>>>(ps, src->stride * PB, (uint8_t*)dst->data, dst->stride * 3, rows,
                                                                          cols, range, table);
    ZB_LAUNCHED();
    t_last_kernel = "colormap";
    return ZB_OK;
}

// Host LUTs, colormaps.zig:92-190, in f64.  @round is half away from zero (std::round); std.math.clamp as @max(lo, @min(v, hi)).
uint8_t round_u8(double v) { return (uint8_t)std::round(v); }
double zig_clamp01(double v) { return std::fmax(0.0, std::fmin(v, 1.0)); }

void jet_eval(double t, uint8_t* rgb) {                                                            // :92-122
    const double gray = 8.0 * t, s = 1.0 / 2.0;
    uint8_t r = 0, g = 0, b = 0;
    if (gray <= 1) { b = round_u8((gray + 1) * s * 255.0); }
    else if (gray <= 3) { g = round_u8((gray - 1) * s * 255.0); b = 255; }
    else if (gray <= 5) { r = round_u8((gray - 3) * s * 255.0); g = 255; b = round_u8((5 - gray) * s * 255.0); }
    else if (gray <= 7) { r = 255; g = round_u8((7 - gray) * s * 255.0); }
    else { r = round_u8((9 - gray) * s * 255.0); }
    rgb[0] = r; rgb[1] = g; rgb[2] = b;
}

void heat_eval(double t, uint8_t* rgb) {                                                           // :133-145
    rgb[0] = round_u8(std::fmin(t / 0.4, 1.0) * 255.0);
    rgb[1] = t > 0.4 ? round_u8(std::fmin((t - 0.4) / 0.4, 1.0) * 255.0) : 0;
    rgb[2] = t > 0.8 ? round_u8(std::fmin((t - 0.8) / 0.2, 1.0) * 255.0) : 0;
}

void turbo_eval(double t, uint8_t* rgb) {                                                          // :156-179
    static const double coeffs[3][6] = {
        {0.13572138, 4.61539260, -42.66032258, 132.13108234, -152.94239396, 59.28637943},
        {0.09140261, 2.19418839, 4.84296658, -14.18503333, 4.27729857, 2.82956604},
        {0.10667330, 12.64194608, -60.58204836, 110.36276771, -89.90310912, 27.34824973}};
    const double t2 = t * t, t3 = t2 * t, t4 = t3 * t, t5 = t4 * t;
    const double v[6] = {1.0, t, t2, t3, t4, t5};
    for (int ch = 0; ch < 3; ++ch) {
        // @reduce(.Add) evaluated left to right (the pairwise order gives the same 768 bytes: tests/test_visual_host.py)
        double acc = v[0] * coeffs[ch][0];
        for (int k = 1; k < 6; ++k) acc = acc + v[k] * coeffs[ch][k];
        rgb[ch] = round_u8(zig_clamp01(acc) * 255.0);
    }
}

// ---- flips and invert ---------------------------------------------------------------------------------------------------------------

// flipLeftRight (transforms.zig:28-33): the block owns pixels [c0, c0 + n) of the left half of row r and their mirror images, and swaps
// the two spans through shared memory.  A middle pixel of an odd width stays.
template <int PB>
__global__ void __launch_bounds__(kThreads) flip_lr_kernel(uint8_t* img, size_t pitch, int rows, int cols) {
    constexpr int P = kSegBytes / PB;
    __shared__ __align__(16) uint8_t sl[kSegBytes + 16], sr[kSegBytes + 16];
    const int r = ZB_GRID_ROW();
    if (r >= rows) return;
    const int half = cols / 2, c0 = blockIdx.x * P, n = min(P, half - c0);
    uint8_t* gl = img + (size_t)r * pitch + (size_t)c0 * PB;
    uint8_t* gr = img + (size_t)r * pitch + (size_t)(cols - c0 - n) * PB;
    uint8_t *ml = shadow(sl, gl), *mr = shadow(sr, gr);
    span_copy<true>(ml, gl, (size_t)n * PB);
    span_copy<true>(mr, gr, (size_t)n * PB);
    __syncthreads();
    for (int j = threadIdx.x; j < n / 2; j += kThreads) {
        swap_bytes<PB>(ml + j * PB, ml + (n - 1 - j) * PB);
        swap_bytes<PB>(mr + j * PB, mr + (n - 1 - j) * PB);
    }
    __syncthreads();
    span_copy<false>(ml, gr, (size_t)n * PB);
    span_copy<false>(mr, gl, (size_t)n * PB);
}

// flipTopBottom (transforms.zig:36-44): the block swaps a segment of row t with the same segment of row rows - 1 - t, t < rows / 2.
template <int PB>
__global__ void __launch_bounds__(kThreads) flip_tb_kernel(uint8_t* img, size_t pitch, int rows, int cols) {
    constexpr int P = kSegBytes / PB;
    __shared__ __align__(16) uint8_t st[kSegBytes + 16], sb[kSegBytes + 16];
    const int t = ZB_GRID_ROW();
    if (t >= rows / 2) return;
    const int c0 = blockIdx.x * P, n = min(P, cols - c0);
    uint8_t* gt = img + (size_t)t * pitch + (size_t)c0 * PB;
    uint8_t* gb = img + (size_t)(rows - 1 - t) * pitch + (size_t)c0 * PB;
    uint8_t *mt = shadow(st, gt), *mb = shadow(sb, gb);
    span_copy<true>(mt, gt, (size_t)n * PB);
    span_copy<true>(mb, gb, (size_t)n * PB);
    __syncthreads();
    span_copy<false>(mt, gb, (size_t)n * PB);
    span_copy<false>(mb, gt, (size_t)n * PB);
}

// invert (image.zig:494-511): 255 - v for u8 components, 1.0 - c for f32 ones (no clamp); Rgba alpha is kept (color.zig:441-444).
template <int F>
__global__ void __launch_bounds__(kThreads) invert_kernel(uint8_t* img, size_t pitch, int rows, int cols) {
    using CT = typename Fmt<F>::CT;
    constexpr int N = Fmt<F>::N, PB = pixel_size<F>(), P = kSegBytes / PB;
    __shared__ __align__(16) uint8_t sm[kSegBytes + 16];
    const int r = ZB_GRID_ROW();
    if (r >= rows) return;
    const int c0 = blockIdx.x * P, n = min(P, cols - c0);
    uint8_t* g = img + (size_t)r * pitch + (size_t)c0 * PB;
    uint8_t* m = shadow(sm, g);
    span_copy<true>(m, g, (size_t)n * PB);
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += kThreads) {
        CT* p = (CT*)(m + j * PB);
#pragma unroll
        for (int k = 0; k < (N == 4 ? 3 : N); ++k) {
            if constexpr (sizeof(CT) == 4) p[k] = __fsub_rn(1.0f, p[k]);
            else p[k] = (CT)(255 - p[k]);
        }
    }
    __syncthreads();
    span_copy<false>(m, g, (size_t)n * PB);
}

bool known_fmt(int pixfmt) { return channels_of(pixfmt) != 0; }
bool shape_eq(const zb_image* a, const zb_image* b) { return a->rows == b->rows && a->cols == b->cols; }
bool empty(const zb_image* a) { return a->rows == 0 || a->cols == 0; }

template <int PB>
int launch_flip(zb_image* img, bool left_right, cudaStream_t s) {
    constexpr int P = kSegBytes / PB;
    const size_t pitch = img->stride * PB;
    const int rows = (int)img->rows, cols = (int)img->cols;
    if (left_right) {
        if (cols < 2) return ZB_OK;
        flip_lr_kernel<PB><<<row_grid(div_up(cols / 2, P), rows), kThreads, 0, s>>>((uint8_t*)img->data, pitch, rows, cols);
    } else {
        if (rows < 2) return ZB_OK;
        flip_tb_kernel<PB><<<row_grid(div_up(cols, P), rows / 2), kThreads, 0, s>>>((uint8_t*)img->data, pitch, rows, cols);
    }
    ZB_LAUNCHED();
    t_last_kernel = left_right ? "flip_left_right" : "flip_top_bottom";
    return ZB_OK;
}

int flip(zb_image* img, int pixfmt, bool left_right, cudaStream_t s) {
    if (!img) return ZB_ERR_INVALID_ARGUMENT;
    if (!known_fmt(pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (empty(img)) return ZB_OK;
    if (!img->data) return ZB_ERR_INVALID_ARGUMENT;
    switch (pixel_bytes(pixfmt)) {
        case 1: return launch_flip<1>(img, left_right, s);
        case 3: return launch_flip<3>(img, left_right, s);
        case 4: return launch_flip<4>(img, left_right, s);
        default: return launch_flip<16>(img, left_right, s);
    }
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_diff(const zb_image* a, const zb_image* b, zb_image* out, int pixfmt, float threshold, float scale, int binary,
                       int force_opaque, zb_diff_stats* stats, zb_stream stream) {
    if (!a || !b || !out) return ZB_ERR_INVALID_ARGUMENT;
    if (!known_fmt(pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (!shape_eq(a, b) || !shape_eq(a, out)) return ZB_ERR_DIMENSION_MISMATCH;                   // diff.zig:34-36
    if (!empty(a) && (!a->data || !b->data || !out->data)) return ZB_ERR_INVALID_ARGUMENT;
    const DiffOpts op{threshold, scale, binary != 0, force_opaque != 0};
    cudaStream_t s = (cudaStream_t)stream;
    switch (pixfmt) {
        case ZB_PIX_U8: return run_diff<ZB_PIX_U8>(a, b, out, op, stats, s);
        case ZB_PIX_F32: return run_diff<ZB_PIX_F32>(a, b, out, op, stats, s);
        case ZB_PIX_RGB8: return run_diff<ZB_PIX_RGB8>(a, b, out, op, stats, s);
        case ZB_PIX_RGBA8: return run_diff<ZB_PIX_RGBA8>(a, b, out, op, stats, s);
        default: return run_diff<ZB_PIX_RGBAF32>(a, b, out, op, stats, s);
    }
}

extern "C" int zb_colormap_lut(int map, uint8_t* lut768) {
    if (!lut768 || map < ZB_COLORMAP_JET || map > ZB_COLORMAP_INFERNO) return ZB_ERR_INVALID_ARGUMENT;
    if (map == ZB_COLORMAP_VIRIDIS || map == ZB_COLORMAP_INFERNO) return ZB_ERR_UNSUPPORTED;      // tables, passed in by the caller
    for (int i = 0; i < 256; ++i) {                                                                // :124-131, :147-154, :182-189
        const double t = (double)i / 255.0;
        if (map == ZB_COLORMAP_JET) jet_eval(t, lut768 + 3 * i);
        else if (map == ZB_COLORMAP_HEAT) heat_eval(t, lut768 + 3 * i);
        else turbo_eval(t, lut768 + 3 * i);
    }
    return ZB_OK;
}

extern "C" int zb_apply_colormap(const zb_image* src, int pixfmt, const uint8_t* lut768, int has_min, double min, int has_max, double max,
                                 zb_image* dst_rgb8, zb_stream stream) {
    if (!src || !lut768 || !dst_rgb8) return ZB_ERR_INVALID_ARGUMENT;
    if (!known_fmt(pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (!shape_eq(src, dst_rgb8)) return ZB_ERR_DIMENSION_MISMATCH;
    if (empty(src)) return ZB_OK;
    if (!src->data || !dst_rgb8->data) return ZB_ERR_INVALID_ARGUMENT;
    Lut768 lut;
    memcpy(lut.v, lut768, sizeof(lut.v));
    cudaStream_t s = (cudaStream_t)stream;
    switch (pixfmt) {
        case ZB_PIX_U8: return run_colormap<ZB_PIX_U8>(src, lut, has_min, min, has_max, max, dst_rgb8, s);
        case ZB_PIX_F32: return run_colormap<ZB_PIX_F32>(src, lut, has_min, min, has_max, max, dst_rgb8, s);
        case ZB_PIX_RGB8: return run_colormap<ZB_PIX_RGB8>(src, lut, has_min, min, has_max, max, dst_rgb8, s);
        case ZB_PIX_RGBA8: return run_colormap<ZB_PIX_RGBA8>(src, lut, has_min, min, has_max, max, dst_rgb8, s);
        default: return run_colormap<ZB_PIX_RGBAF32>(src, lut, has_min, min, has_max, max, dst_rgb8, s);
    }
}

extern "C" int zb_flip_left_right(zb_image* img, int pixfmt, zb_stream s) { return flip(img, pixfmt, true, (cudaStream_t)s); }
extern "C" int zb_flip_top_bottom(zb_image* img, int pixfmt, zb_stream s) { return flip(img, pixfmt, false, (cudaStream_t)s); }

extern "C" int zb_invert(zb_image* img, int pixfmt, zb_stream stream) {
    if (!img) return ZB_ERR_INVALID_ARGUMENT;
    if (!known_fmt(pixfmt) || pixfmt == ZB_PIX_F32) return ZB_ERR_UNSUPPORTED;                    // f32 has no invert (image.zig:510)
    if (empty(img)) return ZB_OK;
    if (!img->data) return ZB_ERR_INVALID_ARGUMENT;
    cudaStream_t s = (cudaStream_t)stream;
    const int rows = (int)img->rows, cols = (int)img->cols;
    uint8_t* p = (uint8_t*)img->data;
    const size_t pitch = img->stride * pixel_bytes(pixfmt);
    const unsigned bx = div_up(cols, kSegBytes / pixel_bytes(pixfmt));
    switch (pixfmt) {
        case ZB_PIX_U8: invert_kernel<ZB_PIX_U8><<<row_grid(bx, rows), kThreads, 0, s>>>(p, pitch, rows, cols); break;
        case ZB_PIX_RGB8: invert_kernel<ZB_PIX_RGB8><<<row_grid(bx, rows), kThreads, 0, s>>>(p, pitch, rows, cols); break;
        case ZB_PIX_RGBA8: invert_kernel<ZB_PIX_RGBA8><<<row_grid(bx, rows), kThreads, 0, s>>>(p, pitch, rows, cols); break;
        default: invert_kernel<ZB_PIX_RGBAF32><<<row_grid(bx, rows), kThreads, 0, s>>>(p, pitch, rows, cols); break;
    }
    ZB_LAUNCHED();
    t_last_kernel = "invert";
    return ZB_OK;
}
