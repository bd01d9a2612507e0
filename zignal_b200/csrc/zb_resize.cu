// zb_resize.cu -- Image.resize.
// Reference: interpolation.zig:89-191 (dispatcher: same-shape copy :91-108; Rgb/Rgba u8 -> integer
// plane resizers; everything else -> resizeGeneric :194-214) and channel_ops.zig:144-493 (plane
// resizers: nearest :193, bilinear :144 (truncating /65536), bicubic :217, Catmull-Rom :292,
// Mitchell :368 (B=C=1/3 hard-coded), Lanczos3 :438 (f32 weights, direct sin, 6x6)).
//
// The plane resizers map destination index d to source s = (d+0.5)*ratio-0.5 in f32 and derive tap
// indices (mirror-resolved) and Q8 / f32 weights from it.  Those per-row and per-column quantities
// depend on one coordinate only, so the host computes them once per call (exactly the reference's
// f32 expressions, including libm sin for Lanczos) and uploads two small tables; the kernel is then
// pure integer (or f32 for Lanczos) accumulate in the reference's ky-outer / kx-inner order.  Pixels
// stay interleaved: the reference's split -> plane -> merge computes the same per-channel values.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <list>
#include <memory>
#include <mutex>
#include <vector>

#include "zb_host_stage.h"
#include "zb_internal.h"
#include "zb_sample.cuh"
#include "zb_warp.h"

namespace zb {

namespace {

struct TapEntry {   // per destination row or column
    int idx[6];     // mirror-resolved source indices
    int w[6];       // Q8 weights (int) or f32 bit patterns (Lanczos); bilinear: w[0] = frac (Q8)
};

// host replicas of the reference's integer kernels ---------------------------------------------
static inline int32_t cubic_q8(int32_t t) {  // channel_ops.zig:228-244
    const int32_t S = 256, at = t < 0 ? -t : t;
    if (at <= S) { const int32_t t2 = (at * at) / S, t3 = (t2 * at) / S; return S - 2 * t2 + t3; }
    if (at <= 2 * S) { const int32_t t2 = (at * at) / S, t3 = (t2 * at) / S; return 4 * S - 8 * at + 5 * t2 - t3; }
    return 0;
}
static inline int32_t catmull_q8(int32_t t) {  // channel_ops.zig:303-319
    const int32_t S = 256, at = t < 0 ? -t : t;
    if (at <= S) { const int32_t t2 = (at * at) / S, t3 = (t2 * at) / S; return S - (5 * t2) / 2 + (3 * t3) / 2; }
    if (at <= 2 * S) { const int32_t t2 = (at * at) / S, t3 = (t2 * at) / S; return 2 * S - 4 * at + (5 * t2) / 2 - t3 / 2; }
    return 0;
}
static inline int32_t mitchell_q8(int32_t t) {  // channel_ops.zig:378-395
    const int64_t s = 256, s2 = s * s, s3 = s2 * s, at = t < 0 ? -(int64_t)t : (int64_t)t;
    if (at < s) { const int64_t a2 = at * at, a3 = a2 * at; return (int32_t)((21 * a3 - 36 * a2 * s + 16 * s3) / (18 * s2)); }
    if (at < 2 * s) { const int64_t a2 = at * at, a3 = a2 * at; return (int32_t)((-7 * a3 + 36 * a2 * s - 60 * at * s2 + 32 * s3) / (18 * s2)); }
    return 0;
}
static inline float lanczos_direct(float x) {  // channel_ops.zig:446-454
    if (x == 0) return 1.0f;
    const float a = 3.0f;
    if (std::fabs(x) >= a) return 0.0f;
    const float pi_x = 3.14159265358979323846f * x;
    return (a * std::sin(pi_x) * std::sin(pi_x / a)) / (pi_x * pi_x);
}
static inline int mirror_idx(long long i, long long n) {  // border.zig:53-60
    if (i >= 0 && i < n) return (int)i;
    if (n == 1) return 0;
    const long long period = 2 * (n - 1);
    long long m = i % period;
    if (m < 0) m += period;
    return (int)(m >= n ? period - m : m);
}

static void build_table(std::vector<TapEntry>& tab, uint32_t src_n, uint32_t dst_n, int method) {
    tab.resize(dst_n);
    const float ratio = (float)src_n / (float)dst_n;
    for (uint32_t d = 0; d < dst_n; ++d) {
        TapEntry e;
        memset(&e, 0, sizeof(e));
        const float sf = ((float)d + 0.5f) * ratio - 0.5f;
        switch (method) {
            case ZB_INTERP_NEAREST: {  // channel_ops.zig:205-206
                const uint32_t v = (uint32_t)std::round(sf);
                e.idx[0] = (int)(v < src_n - 1 ? v : src_n - 1);
                break;
            }
            case ZB_INTERP_BILINEAR: {  // :161-166
                const long long si = (long long)std::floor(sf);
                e.w[0] = (int)std::trunc((sf - std::floor(sf)) * 256.0f);
                e.idx[0] = mirror_idx(si, src_n);
                e.idx[1] = mirror_idx(si + 1, src_n);
                break;
            }
            case ZB_INTERP_BICUBIC:
            case ZB_INTERP_CATMULL_ROM:
            case ZB_INTERP_MITCHELL: {  // :250-272
                const long long si = (long long)std::floor(sf);
                const int32_t f = (int32_t)std::trunc((sf - std::floor(sf)) * 256.0f);
                for (int k = 0; k < 4; ++k) {
                    e.idx[k] = mirror_idx(si + k - 1, src_n);
                    const int32_t t = k * 256 - 256 - f;
                    e.w[k] = method == ZB_INTERP_BICUBIC ? cubic_q8(t) : (method == ZB_INTERP_CATMULL_ROM ? catmull_q8(t) : mitchell_q8(t));
                }
                break;
            }
            default: {  // Lanczos :460-481
                const long long si = (long long)std::floor(sf);
                const float f = sf - std::floor(sf);
                for (int k = 0; k < 6; ++k) {
                    e.idx[k] = mirror_idx(si + k - 2, src_n);
                    const float w = lanczos_direct((float)(k - 2) - f);
                    memcpy(&e.w[k], &w, 4);
                }
                break;
            }
        }
        tab[d] = e;
    }
}

// MODE: 0 nearest, 1 bilinear, 2 4x4 integer cubic family, 3 Lanczos 6x6 f32
template <int CH, int MODE>
__global__ void __launch_bounds__(256) resize_plane_kernel(const uint8_t* __restrict__ src, size_t src_row_b, uint8_t* __restrict__ dst,
                                                           size_t dst_row_b, int dst_rows, int dst_cols,
                                                           const TapEntry* __restrict__ xt, const TapEntry* __restrict__ yt) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = ZB_GRID_ROW();
    if (c >= dst_cols || r >= dst_rows) return;
    const TapEntry ex = xt[c];
    const TapEntry ey = yt[r];
    uint8_t* out = dst + (size_t)r * dst_row_b + (size_t)c * CH;
    if constexpr (MODE == 0) {
        const uint8_t* p = src + (size_t)ey.idx[0] * src_row_b + (size_t)ex.idx[0] * CH;
#pragma unroll
        for (int k = 0; k < CH; ++k) out[k] = p[k];
    } else if constexpr (MODE == 1) {
        const int fx = ex.w[0], fy = ey.w[0];
        const uint8_t* r0 = src + (size_t)ey.idx[0] * src_row_b;
        const uint8_t* r1 = src + (size_t)ey.idx[1] * src_row_b;
#pragma unroll
        for (int k = 0; k < CH; ++k) {
            const int tl = r0[(size_t)ex.idx[0] * CH + k], tr = r0[(size_t)ex.idx[1] * CH + k];
            const int bl = r1[(size_t)ex.idx[0] * CH + k], br = r1[(size_t)ex.idx[1] * CH + k];
            const int top = tl * (256 - fx) + tr * fx;
            const int bottom = bl * (256 - fx) + br * fx;
            const int result = (top * (256 - fy) + bottom * fy) / 65536;  // channel_ops.zig:185, truncating
            out[k] = (uint8_t)(result < 0 ? 0 : (result > 255 ? 255 : result));
        }
    } else if constexpr (MODE == 2) {
        int sum[CH];
#pragma unroll
        for (int k = 0; k < CH; ++k) sum[k] = 0;
        int weight_sum = 0;
#pragma unroll
        for (int ky = 0; ky < 4; ++ky) {
            const uint8_t* row = src + (size_t)ey.idx[ky] * src_row_b;
            const int wy = ey.w[ky];
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) {
                const int w = (ex.w[kx] * wy) / 256;  // @divTrunc(wx * wy, SCALE)
                const uint8_t* p = row + (size_t)ex.idx[kx] * CH;
#pragma unroll
                for (int k = 0; k < CH; ++k) sum[k] += (int)p[k] * w;
                weight_sum += w;
            }
        }
#pragma unroll
        for (int k = 0; k < CH; ++k) {
            const int result = weight_sum != 0 ? sum[k] / weight_sum : 0;
            out[k] = (uint8_t)(result < 0 ? 0 : (result > 255 ? 255 : result));
        }
    } else {
        float sum[CH];
#pragma unroll
        for (int k = 0; k < CH; ++k) sum[k] = 0;
        float weight_sum = 0;
#pragma unroll
        for (int ky = 0; ky < 6; ++ky) {
            const uint8_t* row = src + (size_t)ey.idx[ky] * src_row_b;
            const float wy = __int_as_float(ey.w[ky]);
#pragma unroll
            for (int kx = 0; kx < 6; ++kx) {
                const float w = __int_as_float(ex.w[kx]) * wy;
                const uint8_t* p = row + (size_t)ex.idx[kx] * CH;
#pragma unroll
                for (int k = 0; k < CH; ++k) sum[k] += (float)p[k] * w;
                weight_sum += w;
            }
        }
#pragma unroll
        for (int k = 0; k < CH; ++k) out[k] = clamp_u8_from_float(weight_sum != 0 ? sum[k] / weight_sum : 0.0f);
    }
}

// Cubic family with a UNIFORM phase: when src/dst is an integer ratio every destination column has the same fractional source
// position (frac = 0.5 for even ratios), so the 4 x-weights are the same for all columns, likewise the 4 y-weights for all rows,
// and the 16 products w = @divTrunc(wx * wy, 256) and their sum are per-launch constants instead of 16 multiplies + truncating
// divides and 3 integer divisions by a runtime value per pixel.  Values are identical to the general kernel by construction.
struct UniformCubic {
    int w[16];        // [ky][kx]
    int weight_sum;   // > 0
    float rcp;        // 1 / weight_sum
    int packed[4];    // row ky as four signed bytes (valid when every |w| <= 127): one dp4a does a row of taps
    int dp4a_ok;
};

// four unsigned bytes of a times four signed bytes of b, added to c
__device__ __forceinline__ int dp4a_u8_s8(uint32_t a, int b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

template <int CH>
__global__ void __launch_bounds__(256) resize_cubic_uniform_kernel(const uint8_t* __restrict__ src, size_t src_row_b, size_t src_bytes,
                                                                   uint8_t* __restrict__ dst, size_t dst_row_b, int dst_rows, int dst_cols,
                                                                   const TapEntry* __restrict__ xt, const TapEntry* __restrict__ yt,
                                                                   const __grid_constant__ UniformCubic u) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = ZB_GRID_ROW();
    if (c >= dst_cols || r >= dst_rows) return;
    const int4 ix = __ldg(reinterpret_cast<const int4*>(&xt[c]));   // idx[0..3] lead the entry
    const int4 iy = __ldg(reinterpret_cast<const int4*>(&yt[r]));
    const int iyv[4] = {iy.x, iy.y, iy.z, iy.w};
    int sum[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) sum[k] = 0;
    const bool consecutive = ix.y == ix.x + 1 && ix.z == ix.x + 2 && ix.w == ix.x + 3;   // false only where the mirror border folds
    if (consecutive) {
#pragma unroll
        for (int ky = 0; ky < 4; ++ky) {
            const uint8_t* p = src + (size_t)iyv[ky] * src_row_b + (size_t)ix.x * CH;   // 4 * CH contiguous bytes
            uint32_t wds[CH];                                                            // the 4*CH bytes as CH words
            const uintptr_t a = (uintptr_t)p & 3u;
            const uint32_t* q = reinterpret_cast<const uint32_t*>(p - a);
            if (a == 0) {
#pragma unroll
                for (int i = 0; i < CH; ++i) wds[i] = __ldg(q + i);
            } else if ((const uint8_t*)(q + CH + 1) <= src + src_bytes && (const uint8_t*)q >= src) {
                uint32_t t[CH + 1];
#pragma unroll
                for (int i = 0; i <= CH; ++i) t[i] = __ldg(q + i);
#pragma unroll
                for (int i = 0; i < CH; ++i) wds[i] = __funnelshift_r(t[i], t[i + 1], 8 * (unsigned)a);
            } else {   // the aligned window would leave the image: bytes
#pragma unroll
                for (int i = 0; i < CH; ++i) wds[i] = (uint32_t)p[4 * i] | ((uint32_t)p[4 * i + 1] << 8) | ((uint32_t)p[4 * i + 2] << 16) | ((uint32_t)p[4 * i + 3] << 24);
            }
            if (u.dp4a_ok) {
                // transpose the window to one word per channel (bytes = the 4 taps) and take the row with one dot product:
                // unsigned pixels x signed 8-bit weights, exact in the i32 accumulator
                uint32_t chan[CH];
                if constexpr (CH == 3) {   // r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
                    chan[0] = __byte_perm(__byte_perm(wds[0], wds[1], 0x0630), wds[2], 0x5210);
                    chan[1] = __byte_perm(__byte_perm(wds[0], wds[1], 0x0741), wds[2], 0x6210);
                    chan[2] = __byte_perm(__byte_perm(wds[0], wds[1], 0x0052), wds[2], 0x7410);
                } else {                   // one pixel per word
                    const uint32_t rg01 = __byte_perm(wds[0], wds[1], 0x5140), rg23 = __byte_perm(wds[2], wds[3], 0x5140);
                    const uint32_t ba01 = __byte_perm(wds[0], wds[1], 0x7362), ba23 = __byte_perm(wds[2], wds[3], 0x7362);
                    chan[0] = __byte_perm(rg01, rg23, 0x5410);
                    chan[1] = __byte_perm(rg01, rg23, 0x7632);
                    chan[2] = __byte_perm(ba01, ba23, 0x5410);
                    chan[3] = __byte_perm(ba01, ba23, 0x7632);
                }
#pragma unroll
                for (int k = 0; k < CH; ++k) sum[k] = dp4a_u8_s8(chan[k], u.packed[ky], sum[k]);
            } else {
#pragma unroll
                for (int kx = 0; kx < 4; ++kx)
#pragma unroll
                    for (int k = 0; k < CH; ++k) {
                        const int b = kx * CH + k;
                        sum[k] += (int)((wds[b >> 2] >> (8 * (b & 3))) & 0xFFu) * u.w[ky * 4 + kx];
                    }
            }
        }
    } else {
        const int ixv[4] = {ix.x, ix.y, ix.z, ix.w};
#pragma unroll
        for (int ky = 0; ky < 4; ++ky) {
            const uint8_t* row = src + (size_t)iyv[ky] * src_row_b;
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) {
                const uint8_t* p = row + (size_t)ixv[kx] * CH;
#pragma unroll
                for (int k = 0; k < CH; ++k) sum[k] += (int)p[k] * u.w[ky * 4 + kx];
            }
        }
    }
    uint8_t* out = dst + (size_t)r * dst_row_b + (size_t)c * CH;
#pragma unroll
    for (int k = 0; k < CH; ++k) {
        // @divTrunc(sum, weight_sum) clamped to 0..255: non-positive sums give 0; for positive sums (< 2^24, exact in f32) the
        // float estimate is within one of the quotient and the remainder test fixes it
        int q = 0;
        if (sum[k] > 0) {
            q = __float2int_rz((float)sum[k] * u.rcp);
            const int rem = sum[k] - q * u.weight_sum;
            q += rem >= u.weight_sum ? 1 : (rem < 0 ? -1 : 0);
            q = min(q, 255);
        }
        out[k] = (uint8_t)q;
    }
}

// Exact 4:1 column geometry (idx(c) = 4c + o for every destination column): the four outputs of a lane read 16 CONSECUTIVE source
// pixels, a warp's 128 outputs one contiguous 128*4*CH-byte run per tap row.  The warp fetches that run with fully coalesced
// 128-bit loads (every sector of the source crosses L1 once), parks it in its private shared-memory strip, and each lane picks its
// 4*4*CH bytes back with 128-bit loads (48-byte lane stride: conflict-free).  Taps run on dp4a as above.
template <int CH>
__global__ void __launch_bounds__(CH == 3 ? 256 : 128) resize_cubic_r4_kernel(const uint8_t* __restrict__ src, size_t src_row_b, uint8_t* __restrict__ dst,
                                                              size_t dst_row_b, int dst_rows, int dst_cols, int col_off, size_t src_valid_b, const TapEntry* __restrict__ yt,
                                                              const __grid_constant__ UniformCubic u) {
    constexpr int NW = CH;                 // 16-byte chunks per lane per tap row (4 outputs * 4 taps * CH bytes = 16 * CH)
    constexpr int ROW_BYTES = 32 * NW * 16;
    constexpr int WPB = CH == 3 ? 8 : 4;   // warps per block: 48 KB (Rgb) / 32 KB (Rgba) of strips
    __shared__ __align__(16) uint8_t strip[WPB][4][ROW_BYTES];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = ZB_GRID_ROW();
    const int c_base = (blockIdx.x * WPB + warp) * 128;
    if (c_base >= dst_cols || r >= dst_rows) return;
    const int4 iy = __ldg(reinterpret_cast<const int4*>(&yt[r]));
    const int iyv[4] = {iy.x, iy.y, iy.z, iy.w};
    const size_t run0 = ((size_t)4 * c_base + col_off) * CH;      // first byte of the run inside a source row (multiple of 16)
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
        const uint8_t* rowp = src + (size_t)iyv[ky] * src_row_b;
#pragma unroll
        for (int i = 0; i < NW; ++i) {
            const size_t off = run0 + (size_t)(lane + 32 * i) * 16;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (off + 16 <= src_valid_b) v = __ldg(reinterpret_cast<const uint4*>(rowp + off));   // (row bytes and pitch are multiples of 16)
            *reinterpret_cast<uint4*>(&strip[warp][ky][(lane + 32 * i) * 16]) = v;
        }
    }
    __syncwarp();
    int sum[4][CH];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int k = 0; k < CH; ++k) sum[j][k] = 0;
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
        uint32_t w[4 * NW];
#pragma unroll
        for (int i = 0; i < NW; ++i) {
            const uint4 v = *reinterpret_cast<const uint4*>(&strip[warp][ky][(lane * NW + i) * 16]);
            w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t* wd = w + j * CH;   // the 4 * CH bytes of output j's taps
            uint32_t chan[CH];
            if constexpr (CH == 3) {
                chan[0] = __byte_perm(__byte_perm(wd[0], wd[1], 0x0630), wd[2], 0x5210);
                chan[1] = __byte_perm(__byte_perm(wd[0], wd[1], 0x0741), wd[2], 0x6210);
                chan[2] = __byte_perm(__byte_perm(wd[0], wd[1], 0x0052), wd[2], 0x7410);
            } else {
                const uint32_t rg01 = __byte_perm(wd[0], wd[1], 0x5140), rg23 = __byte_perm(wd[2], wd[3], 0x5140);
                const uint32_t ba01 = __byte_perm(wd[0], wd[1], 0x7362), ba23 = __byte_perm(wd[2], wd[3], 0x7362);
                chan[0] = __byte_perm(rg01, rg23, 0x5410);
                chan[1] = __byte_perm(rg01, rg23, 0x7632);
                chan[2] = __byte_perm(ba01, ba23, 0x5410);
                chan[3] = __byte_perm(ba01, ba23, 0x7632);
            }
#pragma unroll
            for (int k = 0; k < CH; ++k) sum[j][k] = dp4a_u8_s8(chan[k], u.packed[ky], sum[j][k]);
        }
    }
    uint8_t o[4 * CH];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int k = 0; k < CH; ++k) {
            int q = 0;
            const int sv = sum[j][k];
            if (sv > 0) {   // @divTrunc(sum, weight_sum) clamped, as in the kernel above
                q = __float2int_rz((float)sv * u.rcp);
                const int rem = sv - q * u.weight_sum;
                q += rem >= u.weight_sum ? 1 : (rem < 0 ? -1 : 0);
                q = min(q, 255);
            }
            o[j * CH + k] = (uint8_t)q;
        }
    const int c0 = c_base + 4 * lane;
    uint8_t* out = dst + (size_t)r * dst_row_b + (size_t)c0 * CH;
    if (c0 + 4 <= dst_cols && (((uintptr_t)out) & 3u) == 0) {
#pragma unroll
        for (int i = 0; i < CH; ++i)
            reinterpret_cast<uint32_t*>(out)[i] = (uint32_t)o[4 * i] | ((uint32_t)o[4 * i + 1] << 8) | ((uint32_t)o[4 * i + 2] << 16) | ((uint32_t)o[4 * i + 3] << 24);
    } else {
        for (int j = 0; j < 4; ++j)
            if (c0 + j < dst_cols)
                for (int k = 0; k < CH; ++k) out[j * CH + k] = o[j * CH + k];
    }
}

template <int CH>
int launch_plane(const zb_image* src, zb_image* dst, int method, const TapEntry* xt, const TapEntry* yt, cudaStream_t s) {
    const dim3 grid = row_grid(div_up(dst->cols, 256), dst->rows);
    const uint8_t* sp = (const uint8_t*)src->data;
    uint8_t* dp = (uint8_t*)dst->data;
    const size_t sb = (size_t)src->stride * CH, db = (size_t)dst->stride * CH;
    const int dr = (int)dst->rows, dc = (int)dst->cols;
    switch (method) {
        case ZB_INTERP_NEAREST: resize_plane_kernel<CH, 0><<<grid, 256, 0, s>>>(sp, sb, dp, db, dr, dc, xt, yt); break;
        case ZB_INTERP_BILINEAR: resize_plane_kernel<CH, 1><<<grid, 256, 0, s>>>(sp, sb, dp, db, dr, dc, xt, yt); break;
        case ZB_INTERP_LANCZOS: resize_plane_kernel<CH, 3><<<grid, 256, 0, s>>>(sp, sb, dp, db, dr, dc, xt, yt); break;
        default: resize_plane_kernel<CH, 2><<<grid, 256, 0, s>>>(sp, sb, dp, db, dr, dc, xt, yt); break;
    }
    ZB_LAUNCHED();
    return ZB_OK;
}

// resizeGeneric, interpolation.zig:194-214
template <typename CT, int N, int METHOD>
__global__ void __launch_bounds__(256) resize_generic_kernel(SrcView img, CT* __restrict__ dst, size_t dst_stride, int dst_rows,
                                                             int dst_cols, float scale_x, float scale_y, float mb, float mc,
                                                             const float* __restrict__ lut) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = ZB_GRID_ROW();
    if (c >= dst_cols || r >= dst_rows) return;
    const float src_y = ((float)r + 0.5f) * scale_y - 0.5f;
    const float src_x = ((float)c + 0.5f) * scale_x - 0.5f;
    Pix<CT, N> val;
    if (!interpolate<CT, N, METHOD, ZB_BORDER_MIRROR>(img, src_x, src_y, mb, mc, ZB_BORDER_MIRROR, lut, val)) val = zero_px<CT, N>();
    store_px<CT, N>(dst, (size_t)r * dst_stride + c, val);
}

template <typename CT, int N>
int launch_generic(const zb_image* src, zb_image* dst, int method, float mb, float mc, const float* lut, cudaStream_t s) {
    SrcView v{src->data, (int)src->rows, (int)src->cols, src->stride};
    const float scale_x = (float)src->cols / (float)dst->cols;
    const float scale_y = (float)src->rows / (float)dst->rows;
    const dim3 grid = row_grid(div_up(dst->cols, 256), dst->rows);
    return dispatch_method(method, [&](auto m) -> int {
        resize_generic_kernel<CT, N, decltype(m)::value><<<grid, 256, 0, s>>>(v, (CT*)dst->data, (size_t)dst->stride, (int)dst->rows,
                                                                              (int)dst->cols, scale_x, scale_y, mb, mc, lut);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}

// Everything the plane resizers derive from (src shape, dst shape, method), cached per device.  Callers hold a plan by shared_ptr
// from lookup until their launches are queued, so an eviction by another thread cannot free it under them.
struct ResizePlan {
    uint32_t src_rows, src_cols, dst_rows, dst_cols;
    int method, device;
    std::vector<TapEntry> xt, yt;
    TapEntry* dxt = nullptr;   // device copies (one allocation, freed with the plan)
    TapEntry* dyt = nullptr;
    bool uniform_ok = false;   // every row / column has the same cubic weights and the products fit the integer fast path
    bool cols_4to1 = false;    // idx(c) = 4c + o for every column
    UniformCubic u;

    ResizePlan() = default;
    ResizePlan(const ResizePlan&) = delete;
    ResizePlan& operator=(const ResizePlan&) = delete;
    ~ResizePlan() {
        if (!dxt) return;
        // kernels queued on any stream may still read the tables: only the rare eviction pays for this wait
        int cur = 0;
        cudaGetDevice(&cur);
        cudaSetDevice(device);
        cudaDeviceSynchronize();
        cudaFree(dxt);
        cudaSetDevice(cur);
    }
};

int resize_plan(uint32_t src_rows, uint32_t src_cols, uint32_t dst_rows, uint32_t dst_cols, int method, cudaStream_t s,
                std::shared_ptr<const ResizePlan>* out) {
    static std::mutex mu;
    // most recently used first; never destroyed, so no plan frees device memory while the process exits
    static auto* cache = new std::list<std::shared_ptr<const ResizePlan>>();
    int dev = 0;
    ZB_CUDA(cudaGetDevice(&dev));
    std::shared_ptr<const ResizePlan> evicted;   // released after the lock (the last owner's destructor synchronises the device)
    std::lock_guard<std::mutex> lk(mu);
    for (auto it = cache->begin(); it != cache->end(); ++it) {
        const ResizePlan& p = **it;
        if (p.device == dev && p.method == method && p.src_rows == src_rows && p.src_cols == src_cols && p.dst_rows == dst_rows &&
            p.dst_cols == dst_cols) {
            cache->splice(cache->begin(), *cache, it);
            *out = cache->front();
            return ZB_OK;
        }
    }
    auto plp = std::make_shared<ResizePlan>();
    ResizePlan& pl = *plp;
    pl.src_rows = src_rows; pl.src_cols = src_cols; pl.dst_rows = dst_rows; pl.dst_cols = dst_cols;
    pl.method = method; pl.device = dev;
    build_table(pl.xt, src_cols, dst_cols, method);
    build_table(pl.yt, src_rows, dst_rows, method);
    const std::vector<TapEntry>&xt = pl.xt, &yt = pl.yt;
    memset(&pl.u, 0, sizeof(pl.u));
    if (method == ZB_INTERP_BICUBIC || method == ZB_INTERP_CATMULL_ROM || method == ZB_INTERP_MITCHELL) {
        bool uniform = true;
        for (size_t c = 1; c < xt.size() && uniform; ++c) uniform = memcmp(xt[c].w, xt[0].w, 4 * sizeof(int)) == 0;
        for (size_t r = 1; r < yt.size() && uniform; ++r) uniform = memcmp(yt[r].w, yt[0].w, 4 * sizeof(int)) == 0;
        UniformCubic& u = pl.u;
        u.weight_sum = 0;
        for (int ky = 0; ky < 4; ++ky)
            for (int kx = 0; kx < 4; ++kx) {
                u.w[ky * 4 + kx] = (xt[0].w[kx] * yt[0].w[ky]) / 256;   // @divTrunc(wx * wy, SCALE), channel_ops.zig:262
                u.weight_sum += u.w[ky * 4 + kx];
            }
        long long abs_sum = 0;
        for (int i = 0; i < 16; ++i) abs_sum += std::llabs((long long)u.w[i]);
        if (uniform && u.weight_sum > 0 && 255 * abs_sum < (1 << 24)) {
            pl.uniform_ok = true;
            u.rcp = 1.0f / (float)u.weight_sum;
            u.dp4a_ok = 1;
            for (int i = 0; i < 16; ++i) u.dp4a_ok &= (u.w[i] >= -128 && u.w[i] <= 127) ? 1 : 0;
            for (int ky = 0; ky < 4; ++ky) {
                uint32_t pk = 0;
                for (int kx = 0; kx < 4; ++kx) pk |= ((uint32_t)(u.w[ky * 4 + kx] & 0xFF)) << (8 * kx);
                u.packed[ky] = (int)pk;
            }
            bool r4 = true;
            const int o = xt[0].idx[0];
            for (size_t c = 0; c < xt.size() && r4; ++c)
                for (int k = 0; k < 4; ++k) r4 = r4 && xt[c].idx[k] == (int)(4 * c) + o + k;
            pl.cols_4to1 = r4;
        }
    }
    // one device allocation for both tables, uploaded once per plan on the caller's stream and synchronised before the plan enters
    // the cache (any stream may use it afterwards).  On failure the plan's destructor frees the allocation.
    const size_t nx = xt.size(), ny = yt.size();
    ZB_CUDA(cudaMalloc(&pl.dxt, (nx + ny) * sizeof(TapEntry)));
    pl.dyt = pl.dxt + nx;
    ZB_CUDA(cudaMemcpyAsync(pl.dxt, xt.data(), nx * sizeof(TapEntry), cudaMemcpyHostToDevice, s));
    ZB_CUDA(cudaMemcpyAsync(pl.dyt, yt.data(), ny * sizeof(TapEntry), cudaMemcpyHostToDevice, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    if (cache->size() >= 32) {   // evict the least recently used plan; it is freed when its last user lets go of it
        evicted = std::move(cache->back());
        cache->pop_back();
    }
    cache->push_front(std::move(plp));
    *out = cache->front();
    return ZB_OK;
}

}  // namespace

int resize_dispatch(const zb_image* src, zb_image* dst, int pixfmt, int method, float mb, float mc, cudaStream_t s) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (!pixfmt_in(kFmtAll, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (method < ZB_INTERP_NEAREST || method > ZB_INTERP_LANCZOS) return ZB_ERR_INVALID_ARGUMENT;
    if (src->rows == dst->rows && src->cols == dst->cols) return zb_copy(src, dst, pixfmt, (zb_stream)s);  // :91-108
    if (exceeds_int_index(src, pixfmt) || exceeds_int_index(dst, pixfmt)) return ZB_ERR_UNSUPPORTED;
    if (dst->rows == 0 || dst->cols == 0) return ZB_OK;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (src->rows == 0 || src->cols == 0) {  // every sample is null -> zeroes (:205-210)
        return span_zero(dst->data, dst->stride * pixel_bytes(pixfmt), (size_t)dst->cols * pixel_bytes(pixfmt), dst->rows, s);
    }
    return dispatch_pixfmt<kFmtAll>(pixfmt, [&](auto f) -> int {
        using P = Fmt<decltype(f)::value>;
        constexpr int ch = P::N;
        if constexpr (std::is_same_v<typename P::CT, uint8_t> && ch > 1) {  // meta.isRgb(T), :111
            // tap tables and everything derived from them depend only on (src shape, dst shape, method): built once per device,
            // kept in device memory (the per-call rebuild + two pageable uploads cost more than the 4:1 kernel itself)
            std::shared_ptr<const ResizePlan> plan;   // held until the launches below are queued
            if ((rc = resize_plan(src->rows, src->cols, dst->rows, dst->cols, method, s, &plan))) return rc;
            const std::vector<TapEntry>& xt = plan->xt;
            const TapEntry* dxt = plan->dxt;
            const TapEntry* dyt = plan->dyt;
            if (method == ZB_INTERP_BICUBIC || method == ZB_INTERP_CATMULL_ROM || method == ZB_INTERP_MITCHELL) {
                const UniformCubic& u = plan->u;
                if (plan->uniform_ok) {
                    const dim3 grid = row_grid(div_up(dst->cols, 256), dst->rows);
                    const size_t sb = (size_t)src->stride * ch, db = (size_t)dst->stride * ch;
                    const size_t src_bytes = (size_t)(src->rows - 1) * sb + (size_t)src->cols * ch;
                    // exact 4:1 columns: idx(c) = 4c + o for every column, 16-byte friendly addresses -> the coalesced strip kernel
                    const size_t valid_b = (size_t)src->cols * ch;
                    bool r4 = u.dp4a_ok && ((uintptr_t)src->data & 15u) == 0 && sb % 16 == 0 && valid_b % 16 == 0;
                    const int o = xt[0].idx[0];
                    r4 = r4 && plan->cols_4to1 && o >= 0 && ((size_t)o * ch) % 16 == 0;
                    if (r4) {
                        const dim3 g4 = row_grid(div_up(dst->cols, ch == 3 ? 1024 : 512), dst->rows);
                        resize_cubic_r4_kernel<ch><<<g4, ch == 3 ? 256 : 128, 0, s>>>((const uint8_t*)src->data, sb, (uint8_t*)dst->data, db,
                                                                                      (int)dst->rows, (int)dst->cols, o, valid_b, dyt, u);
                        ZB_LAUNCHED();
                        t_last_kernel = "resize_cubic_r4_u8";
                        return ZB_OK;
                    }
                    resize_cubic_uniform_kernel<ch><<<grid, 256, 0, s>>>((const uint8_t*)src->data, sb, src_bytes, (uint8_t*)dst->data, db,
                                                                         (int)dst->rows, (int)dst->cols, dxt, dyt, u);
                    ZB_LAUNCHED();
                    t_last_kernel = "resize_cubic_uniform_u8";
                    return ZB_OK;
                }
            }
            t_last_kernel = "resize_plane_u8";
            return launch_plane<ch>(src, dst, method, dxt, dyt, s);
        } else {
            const float* lut = nullptr;
            if (method == ZB_INTERP_LANCZOS && (rc = lanczos_lut_device(&lut, s))) return rc;
            t_last_kernel = "resize_generic";
            return launch_generic<typename P::CT, ch>(src, dst, method, mb, mc, lut, s);
        }
    });
}

}  // namespace zb

using namespace zb;

extern "C" {

int zb_resize(const zb_image* src, zb_image* dst, int pixfmt, int method, float mb, float mc, zb_stream s) {
    return resize_dispatch(src, dst, pixfmt, method, mb, mc, (cudaStream_t)s);
}

int zb_host_resize(const zb_image* src, zb_image* dst, int pixfmt, int method, float mb, float mc) {
    if (!src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    HostStage st;
    int rc;
    if ((rc = st.begin(src, dst, pixfmt))) return rc;
    if ((rc = resize_dispatch(&st.dsrc, &st.ddst, pixfmt, method, mb, mc, st.stream))) return rc;
    return st.finish(dst, pixfmt);
}

}  // extern "C"
