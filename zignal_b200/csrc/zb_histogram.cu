// zb_histogram.cu -- Image.histogram / autocontrast / equalize / thresholdOtsu on 8-bit images (U8, RGB8, RGBA8).
//
// Reference: image.zig:1161-1185 (histogram over the pixel iterator, u32 counts per channel, alpha included),
// image/histogram.zig:123-162 (findCutoffMin / findCutoffMax), image/enhancement.zig:11-80 (autocontrast), :84-252 (equalize),
// image/binary.zig:38-84 (thresholdOtsu).
//
// Two launches per operation, no host round trip in between:
//   hist_kernel : 16-byte loads (scalar head / tail where a row is not 16-byte aligned), one sub-histogram per warp in shared
//                 memory, merged into global u32 counts once per CTA.  A lane whose 16 bytes are one repeated pixel joins the
//                 lanes holding the same pixel (__match_any_sync) and their leader adds the whole group at once, so a constant
//                 image does not serialise 32 lanes on one shared-memory bin.  The last CTA to finish (ticket) builds the
//                 256-entry-per-channel table: the autocontrast / equalize remap, or Otsu's threshold and its 0 / 255 map.
//   lut_kernel  : applies the table (in shared memory) to 16 bytes per thread; RGB8 takes the byte's channel modulo 3.
// The table arithmetic follows the reference operation by operation (explicit _rn intrinsics), with one documented deviation:
// equalize forms (cdf[i] - cdf_min) * 255 in 64 bits.  The reference's u32 product overflows once total - cdf_min exceeds
// 16,843,009 (e.g. any 8192 x 8192 image), where Zig traps (safe builds) or is undefined (ReleaseFast); the 64-bit product is the
// value the formula intends.
// Images of 2^32 pixels or more return ZB_ERR_UNSUPPORTED: the reference's u32 counts and rows * cols would wrap.
#include <algorithm>
#include <cmath>

#include "zb_internal.h"

namespace zb {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr long long kSeg = (long long)kThreads * 16 * 4;   // bytes of a row one CTA takes per work item

enum { MODE_COUNT = 0, MODE_AUTOCONTRAST = 1, MODE_EQUALIZE = 2, MODE_OTSU = 3 };

// Scratch layout of one call (zeroed before the histogram kernel).
struct HistState {
    uint32_t counts[4 * 256];
    uint32_t ticket;
    uint32_t threshold;   // Otsu
    uint8_t lut[4 * 256];
};

struct Walk {               // rows of bytes, split into work items of kSeg bytes
    long long rows, row_bytes, n_seg;
    size_t src_pitch, dst_pitch;
};

struct HistParams {
    const uint8_t* src;
    Walk w;
    HistState* st;
    int mode;
    uint32_t total;           // rows * cols
    uint32_t cutoff_pixels;   // autocontrast
};

// ---- histogram ------------------------------------------------------------------------------------------------------------------
template <int CH>
__device__ __forceinline__ void add_chunk(uint32_t (*h)[256], uint4 v, int phase, bool valid) {
    // is the chunk one repeated pixel?  (16 bytes periodic with the pixel size; the key also carries the channel phase)
    bool uni;
    unsigned long long key;
    if constexpr (CH == 1) {
        const uint32_t rep = (v.x & 0xFFu) * 0x01010101u;
        uni = v.x == rep && v.y == rep && v.z == rep && v.w == rep;
        key = v.x & 0xFFu;
    } else if constexpr (CH == 4) {
        uni = v.x == v.y && v.x == v.z && v.x == v.w;
        key = (unsigned long long)v.x | ((unsigned long long)phase << 32);
    } else {
        uni = __funnelshift_r(v.x, v.y, 24) == v.x && __funnelshift_r(v.y, v.z, 24) == v.y && __funnelshift_r(v.z, v.w, 24) == v.z &&
              (v.w >> 24) == (v.w & 0xFFu);
        key = (unsigned long long)(v.x & 0xFFFFFFu) | ((unsigned long long)phase << 32);
    }
    const int lane = threadIdx.x & 31;
    uni = uni && valid;
    if (!uni) key = (1ull << 40) | (unsigned long long)lane;   // a key no other lane has
    const unsigned group = __match_any_sync(0xffffffffu, key);
    if (uni) {
        if (lane == __ffs(group) - 1) {
            const uint32_t n = __popc(group);
            const uint32_t b[4] = {v.x & 0xFFu, (v.x >> 8) & 0xFFu, (v.x >> 16) & 0xFFu, v.x >> 24};
#pragma unroll
            for (int j = 0; j < CH; ++j) {   // byte j of the chunk: channel (phase + j) % CH, 16 / CH bytes (RGB: 6, 5, 5 from j)
                const int ch = (phase + j) % CH;
                const uint32_t bytes = CH == 3 ? (j == 0 ? 6u : 5u) : 16u / CH;
                atomicAdd(&h[ch][b[j]], n * bytes);
            }
        }
    } else if (valid) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        int ch = phase;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            atomicAdd(&h[CH == 1 ? 0 : ch][(w[j >> 2] >> (8 * (j & 3))) & 0xFFu], 1u);
            if (CH > 1) ch = ch + 1 == CH ? 0 : ch + 1;
        }
    }
}

template <int CH>
__device__ void build_table(const HistParams& p);

template <int CH>
__global__ void __launch_bounds__(kThreads) hist_kernel(const HistParams p) {
    __shared__ uint32_t sh[kWarps][CH][256];
    __shared__ bool is_last;
    for (int i = threadIdx.x; i < kWarps * CH * 256; i += kThreads) (&sh[0][0][0])[i] = 0u;
    __syncthreads();
    uint32_t (*h)[256] = sh[threadIdx.x >> 5];
    const long long n_work = p.w.rows * p.w.n_seg;
    for (long long wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
        const long long r = wi / p.w.n_seg;
        const long long s0 = (wi - r * p.w.n_seg) * kSeg, s1 = min(p.w.row_bytes, s0 + kSeg);
        const uint8_t* rowp = p.src + (size_t)r * p.w.src_pitch;
        const long long a0 = min(s1, s0 + (long long)((16u - ((uintptr_t)(rowp + s0) & 15u)) & 15u));
        const long long a1 = a0 + ((s1 - a0) & ~15ll);
        for (long long o = s0 + threadIdx.x; o < a0; o += kThreads) atomicAdd(&h[CH == 1 ? 0 : (int)(o % CH)][rowp[o]], 1u);
        for (long long o = a1 + threadIdx.x; o < s1; o += kThreads) atomicAdd(&h[CH == 1 ? 0 : (int)(o % CH)][rowp[o]], 1u);
        const int phase = CH == 1 ? 0 : (int)(a0 % CH);   // 16 is 1 mod 3 and 0 mod 4: the phase of chunk k is (phase + k) % CH
        for (long long base = a0; base < a1; base += 16ll * kThreads) {   // block-uniform trip count: full warps at the match
            const long long o = base + 16ll * threadIdx.x;
            const bool valid = o < a1;
            const uint4 v = valid ? __ldg(reinterpret_cast<const uint4*>(rowp + o)) : make_uint4(0, 0, 0, 0);
            add_chunk<CH>(h, v, CH == 3 ? (int)((phase + (o - a0) / 16) % 3) : phase, valid);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < CH * 256; i += kThreads) {
        uint32_t s = 0;
#pragma unroll
        for (int k = 0; k < kWarps; ++k) s += (&sh[k][0][0])[i];
        if (s) atomicAdd(&p.st->counts[i], s);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        is_last = atomicAdd(&p.st->ticket, 1u) == gridDim.x - 1u;
    }
    __syncthreads();
    if (is_last && p.mode != MODE_COUNT) {
        __threadfence();
        build_table<CH>(p);
    }
}

// The table of the last CTA.  Integer prefix sums are exact in any order; the f32 / f64 steps follow the reference one by one.
template <int CH>
__device__ void build_table(const HistParams& p) {
    __shared__ uint32_t cnt[CH][256];
    __shared__ uint32_t lo[CH], hi[CH];
    for (int i = threadIdx.x; i < CH * 256; i += kThreads) (&cnt[0][0])[i] = __ldcg(&p.st->counts[i]);
    __syncthreads();
    const int t = threadIdx.x;
    if (p.mode == MODE_AUTOCONTRAST) {
        if (t < CH) {   // findCutoffMin / findCutoffMax, histogram.zig:123-162
            const uint32_t* v = cnt[t];
            const uint32_t cut = p.cutoff_pixels;
            uint32_t mn = 0, mx = 0;
            if (cut == 0) {
                mn = 0;
                for (int i = 0; i < 256; ++i) if (v[i] > 0) { mn = i; break; }
                mx = 0;
                for (int i = 255; i > 0; --i) if (v[i] > 0) { mx = i; break; }   // `while (i > 0)`: bin 0 is never visited
            } else {
                uint32_t cum = 0;
                mn = 255;
                for (int i = 0; i < 256; ++i) { cum += v[i]; if (cum > cut) { mn = i; break; } }
                cum = 0;
                mx = 0;
                for (int i = 255; i > 0; --i) { cum += v[i]; if (cum > cut) { mx = i; break; } }
            }
            lo[t] = mn;
            hi[t] = mx;
        }
        __syncthreads();
        for (int i = t; i < CH * 256; i += kThreads) {   // enhancement.zig:35-40 / :58-63, per channel; Rgba alpha is left as it is
            const int ch = i >> 8, val = i & 255;
            uint8_t out = (uint8_t)val;
            if (!(CH == 4 && ch == 3)) {
                const int mn = (int)lo[ch], mx = (int)hi[ch];
                const int clamped = max(mn, min(mx, val));                // @max(min, @min(max, v)): min when max < min
                const int range = mx > mn ? mx - mn : 1;
                const float normalized = __fdiv_rn((float)(clamped - mn), (float)range);
                out = (uint8_t)roundf(__fmul_rn(normalized, 255.0f));     // @round: half away from zero; the value lies in [0, 255]
            }
            p.st->lut[i] = out;
        }
    } else if (p.mode == MODE_EQUALIZE) {
        __shared__ uint32_t cdf[CH][256];
        if (t < CH) {
            uint32_t run = 0, first = 0;
            for (int i = 0; i < 256; ++i) {
                run += cnt[t][i];
                cdf[t][i] = run;
                if (first == 0 && run > 0) first = run;   // cdf_min: the first non-zero CDF value
            }
            lo[t] = first;
        }
        __syncthreads();
        for (int i = t; i < CH * 256; i += kThreads) {   // enhancement.zig:112-127 / :210-229; Rgba alpha is equalized as well
            const int ch = i >> 8, val = i & 255;
            const uint32_t cdf_min = lo[ch];
            const uint32_t den = p.total - cdf_min;
            uint8_t out;
            if (den == 0) out = (uint8_t)val;
            else if (cdf[ch][val] >= cdf_min) out = (uint8_t)(((uint64_t)(cdf[ch][val] - cdf_min) * 255u) / den);   // 64-bit numerator
            else out = 0;
            p.st->lut[i] = out;
        }
    } else {   // MODE_OTSU (u8 only), binary.zig:38-84
        __shared__ unsigned long long cum_n[256], cum_s[256];
        __shared__ double best_v[kWarps];
        __shared__ int best_i[kWarps];
        if (t == 0) {   // weight_background and sum_background are integers below 2^53: the f64 running sums are these, exactly
            unsigned long long n = 0, s = 0;
            for (int i = 0; i < 256; ++i) {
                n += cnt[0][i];
                s += (unsigned long long)cnt[0][i] * (unsigned long long)i;
                cum_n[i] = n;
                cum_s[i] = s;
            }
        }
        __syncthreads();
        const double total = (double)p.total;
        const double sum_total = (double)cum_s[255];
        double var = -1.0;
        const double wb = (double)cum_n[t];
        const double wf = __dsub_rn(total, wb);
        // `continue` while weight_background == 0, `break` at the first weight_foreground == 0 (every later bin has it too)
        const bool cand = wb != 0.0 && wf != 0.0;
        if (cand) {
            const double sb = (double)cum_s[t];
            const double mean_b = __ddiv_rn(sb, wb);
            const double mean_f = __ddiv_rn(__dsub_rn(sum_total, sb), wf);
            const double diff = __dsub_rn(mean_b, mean_f);
            var = __dmul_rn(__dmul_rn(__dmul_rn(wb, wf), diff), diff);   // wb * wf * diff * diff, left to right
        }
        // first index of the maximum (strict `variance > max_variance` from -1 keeps the earliest bin on ties)
        int bi = cand ? t : 256;
        double bv = var;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const double ov = __shfl_down_sync(0xffffffffu, bv, d);
            const int oi = __shfl_down_sync(0xffffffffu, bi, d);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if ((t & 31) == 0) { best_v[t >> 5] = bv; best_i[t >> 5] = bi; }
        __syncthreads();
        if (t == 0) {
            double v = best_v[0];
            int idx = best_i[0];
            for (int k = 1; k < kWarps; ++k)
                if (best_v[k] > v || (best_v[k] == v && best_i[k] < idx)) { v = best_v[k]; idx = best_i[k]; }
            lo[0] = idx < 256 ? (uint32_t)idx : 0u;   // no candidate bin: threshold stays 0
            p.st->threshold = lo[0];
        }
        __syncthreads();
        p.st->lut[t] = t > (int)lo[0] ? 255 : 0;   // src > t ? 255 : 0 (binary.zig:77-82)
    }
}

// ---- table map ----------------------------------------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(kThreads) lut_kernel(const uint8_t* src, uint8_t* dst, const Walk w, const uint8_t* lut_g) {
    __shared__ uint8_t lut[CH * 256];
    for (int i = threadIdx.x; i < CH * 256; i += kThreads) lut[i] = lut_g[i];
    __syncthreads();
    const long long n_work = w.rows * w.n_seg;
    for (long long wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
        const long long r = wi / w.n_seg;
        const long long s0 = (wi - r * w.n_seg) * kSeg;
        const int n = (int)min(w.row_bytes - s0, kSeg);           // bytes of this work item
        const uint8_t* sp = src + (size_t)r * w.src_pitch + s0;
        uint8_t* dp = dst + (size_t)r * w.dst_pitch + s0;
        const int ph = CH == 1 ? 0 : (int)(s0 % CH);              // channel of byte 0
        auto map1 = [&](int o) { dp[o] = lut[CH == 1 ? sp[o] : ((ph + o) % CH) * 256 + sp[o]]; };
        if ((((uintptr_t)sp ^ (uintptr_t)dp) & 15u) != 0) {   // source and destination rows not co-aligned: bytes
            for (int o = threadIdx.x; o < n; o += kThreads) map1(o);
            continue;
        }
        const int a0 = min(n, (int)((16u - ((uintptr_t)sp & 15u)) & 15u));
        const int a1 = a0 + ((n - a0) & ~15);
        for (int o = threadIdx.x; o < a0; o += kThreads) map1(o);
        for (int o = a1 + threadIdx.x; o < n; o += kThreads) map1(o);
        for (int o = a0 + 16 * threadIdx.x; o < a1; o += 16 * kThreads) {
            const uint4 v = *reinterpret_cast<const uint4*>(sp + o);
            int ch = CH == 1 ? 0 : (ph + o) % CH;
            auto map4 = [&](uint32_t x) {
                uint32_t word = 0;
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    word |= (uint32_t)lut[ch * 256 + ((x >> (8 * b)) & 0xFFu)] << (8 * b);
                    if (CH > 1) ch = ch + 1 == CH ? 0 : ch + 1;
                }
                return word;
            };
            const uint32_t ox = map4(v.x), oy = map4(v.y), oz = map4(v.z), ow = map4(v.w);
            *reinterpret_cast<uint4*>(dp + o) = make_uint4(ox, oy, oz, ow);
        }
    }
}

// Rows of bytes; a contiguous image (or a pair of them) is walked as one long row so that tall, narrow images still fill the GPU.
Walk make_walk(const zb_image* src, const zb_image* dst, int ch) {
    Walk w;
    const size_t rb = (size_t)src->cols * ch;
    w.src_pitch = (size_t)src->stride * ch;
    w.dst_pitch = dst ? (size_t)dst->stride * ch : w.src_pitch;
    w.rows = src->rows;
    w.row_bytes = (long long)rb;
    if (w.src_pitch == rb && w.dst_pitch == rb) {
        w.row_bytes = (long long)rb * src->rows;
        w.rows = 1;
    }
    w.n_seg = (w.row_bytes + kSeg - 1) / kSeg;
    return w;
}

// Queue the histogram (and the table of `mode`) of src into a zeroed HistState.
int run_hist(const zb_image* src, int pixfmt, int mode, uint32_t cutoff_pixels, HistState* st, cudaStream_t s) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    ZB_CUDA(cudaMemsetAsync(st, 0, sizeof(HistState), s));
    HistParams p;
    p.src = (const uint8_t*)src->data;
    p.w = make_walk(src, nullptr, channels_of(pixfmt));
    p.st = st;
    p.mode = mode;
    p.total = (uint32_t)((uint64_t)src->rows * src->cols);
    p.cutoff_pixels = cutoff_pixels;
    const long long n_work = p.w.rows * p.w.n_seg;
    // as many CTAs as fit at once: the loads of every resident thread are what keeps HBM busy
    auto launch = [&](auto kernel) -> int {
        int per_sm = 1;
        ZB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0));
        const unsigned grid = (unsigned)std::min<long long>(n_work, (long long)std::max(per_sm, 1) * di.sm_count);
        kernel<<<grid, kThreads, 0, s>>>(p);
        return ZB_OK;
    };
    rc = dispatch_pixfmt<kFmt8Bit>(pixfmt, [&](auto f) -> int { return launch(hist_kernel<Fmt<decltype(f)::value>::N>); });
    if (rc) return rc;
    ZB_LAUNCHED();
    return ZB_OK;
}

int run_lut(const zb_image* src, zb_image* dst, int pixfmt, const uint8_t* lut, cudaStream_t s) {
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const Walk w = make_walk(src, dst, channels_of(pixfmt));
    const long long n_work = w.rows * w.n_seg;
    const unsigned grid = (unsigned)std::min<long long>(n_work, 8ll * di.sm_count);   // 8 x 256 threads fill an SM
    const uint8_t* sp = (const uint8_t*)src->data;
    uint8_t* dp = (uint8_t*)dst->data;
    return dispatch_pixfmt<kFmt8Bit>(pixfmt, [&](auto f) -> int {
        lut_kernel<Fmt<decltype(f)::value>::N><<<grid, kThreads, 0, s>>>(sp, dp, w, lut);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}

bool too_many_pixels(const zb_image* img) { return (uint64_t)img->rows * img->cols >= (1ull << 32); }

// autocontrast / equalize: histogram + table, then the map in place.
int enhance(zb_image* img, int pixfmt, int mode, uint32_t cutoff_pixels, cudaStream_t s) {
    Scratch st;
    int rc = st.alloc(sizeof(HistState), s);
    if (rc) return rc;
    if ((rc = run_hist(img, pixfmt, mode, cutoff_pixels, st.as<HistState>(), s))) return rc;
    if ((rc = run_lut(img, img, pixfmt, st.as<HistState>()->lut, s))) return rc;
    t_last_kernel = mode == MODE_EQUALIZE ? "equalize" : "autocontrast";
    return ZB_OK;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" {

int zb_histogram(const zb_image* src, int pixfmt, uint32_t* counts, zb_stream stream) {
    if (!src || !counts) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmt8Bit, pixfmt)) return ZB_ERR_UNSUPPORTED;   // image.zig:1181
    if (too_many_pixels(src)) return ZB_ERR_UNSUPPORTED;
    const int ch = channels_of(pixfmt);
    if (src->rows == 0 || src->cols == 0) {
        memset(counts, 0, (size_t)ch * 256 * sizeof(uint32_t));
        return ZB_OK;
    }
    cudaStream_t s = (cudaStream_t)stream;
    Scratch st;
    int rc = st.alloc(sizeof(HistState), s);
    if (rc) return rc;
    if ((rc = run_hist(src, pixfmt, MODE_COUNT, 0, st.as<HistState>(), s))) return rc;
    ZB_CUDA(cudaMemcpyAsync(counts, st.as<HistState>()->counts, (size_t)ch * 256 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    t_last_kernel = "histogram";
    return ZB_OK;
}

int zb_autocontrast(zb_image* img, int pixfmt, float cutoff, zb_stream stream) {
    if (!img) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmt8Bit, pixfmt)) return ZB_ERR_UNSUPPORTED;                    // enhancement.zig:75,78
    if (!(cutoff >= 0.0f && cutoff < 0.5f)) return ZB_ERR_INVALID_CUTOFF;  // :16-18 (NaN, which the reference cannot convert, too)
    if (too_many_pixels(img)) return ZB_ERR_UNSUPPORTED;
    if (img->rows == 0 || img->cols == 0) return ZB_OK;
    const float prod = (float)((uint64_t)img->rows * img->cols) * cutoff;   // :21 @trunc(f32(total) * cutoff)
    const uint32_t cutoff_pixels = (uint32_t)std::trunc(prod);
    return enhance(img, pixfmt, MODE_AUTOCONTRAST, cutoff_pixels, (cudaStream_t)stream);
}

int zb_equalize(zb_image* img, int pixfmt, zb_stream stream) {
    if (!img) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmt8Bit, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (too_many_pixels(img)) return ZB_ERR_UNSUPPORTED;                 // enhancement.zig:85 @intCast to u32
    if (img->rows == 0 || img->cols == 0) return ZB_OK;
    return enhance(img, pixfmt, MODE_EQUALIZE, 0, (cudaStream_t)stream);
}

int zb_threshold_otsu(const zb_image* src, zb_image* dst, uint8_t* threshold, zb_stream stream) {
    if (!src || !dst || !threshold) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZB_ERR_DIMENSION_MISMATCH;   // image.zig:849
    if (src->rows == 0 || src->cols == 0) { *threshold = 0; return ZB_OK; }                 // binary.zig:39-41: out untouched
    if (too_many_pixels(src)) return ZB_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch st, tmp;
    int rc = st.alloc(sizeof(HistState), s);
    if (rc) return rc;
    HistState* hs = st.as<HistState>();
    zb_image in = *src;
    // the map reads and writes each byte in one thread, so only a shifted overlap needs a snapshot of the source
    if (images_overlap(src, dst, 1) && !(src->data == dst->data && src->stride == dst->stride)) {
        if ((rc = tmp.alloc((size_t)src->rows * src->cols, s))) return rc;
        in.data = tmp.p;
        in.stride = src->cols;
        if ((rc = zb_copy(src, &in, ZB_PIX_U8, stream))) return rc;
    }
    if ((rc = run_hist(&in, ZB_PIX_U8, MODE_OTSU, 0, hs, s))) return rc;
    if ((rc = run_lut(&in, dst, ZB_PIX_U8, hs->lut, s))) return rc;
    uint32_t t = 0;
    ZB_CUDA(cudaMemcpyAsync(&t, &hs->threshold, sizeof(t), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    *threshold = (uint8_t)t;
    t_last_kernel = "threshold_otsu";
    return ZB_OK;
}

}  // extern "C"
