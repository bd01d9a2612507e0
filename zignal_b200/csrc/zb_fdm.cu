// zb_fdm.cu -- FeatureDistributionMatching (reference fdm.zig:19-275) on the device.
//
// The reference makes two sequential full passes per image: a Welford mean/co-moment stream
// (stats.zig:261-280, a ~10-flop dependency chain per pixel) and the per-pixel affine colour map.
// Here the statistics pass is a parallel reduction of EXACT integer moments of the u8 pixels
// (n, sum x_i, sum x_i x_j as u64; integer atomics, so the result is order-independent), finished in
// f64: cov_ij = (n*Sij - Si*Sj) / (n (n-1) 255^2) with the numerator exact in 128 bits.
// That differs from Welford only by Welford's own rounding noise (~1e-16 relative).  The 3x3 SVDs,
// W = Us * diag(sqrt(lt/ls)) * Ut^T and the bias follow fdm.zig:199-254 verbatim in f64.  For `update` that
// small solve runs ON THE DEVICE in a one-thread kernel between the two passes (same source as the host
// version, zb_svd_core.h: + - * / sqrt only, so the bits are the same) -- no device-to-host round trip, the
// three kernels are simply queued on the stream.  The map (fdm.zig:257-271) is one f64 kernel:
// res = r*w0 + g*w1 + b*w2 + bias, round(255*clamp(res,0,1)).
// The 11 moment sums are also the quantities one all-reduce combines when an image is sharded
// across GPUs (zb_fdm_moments / zb_fdm_update_with_moments).
#include <cmath>
#include <cstring>

#include "zb_host_stage.h"
#include "zb_internal.h"
#include "zb_linalg.h"
#include "zb_shard.h"
#include "zb_svd_core.h"

struct FdmTarget {   // what `update` needs from the target (fdm.zig:92-121)
    double mean[3];
    double u[9];
    double s[3];
    int is_gray;
};

struct zb_fdm {
    int pixfmt;
    double target_mean[3];
    double target_u[9];
    double target_s[3];
    bool target_is_gray;
    bool has_target, has_source;
    zb_image source;
    // device side of `update`: the 11 moment sums, the solved map parameters, a status word (0 or ZB_ERR_NOT_CONVERGED)
    unsigned long long* d_m;
    void* d_params;
    int* d_status;
};

namespace zb {
namespace {

// color.zig:1031-1041 rgbToGray(u8)
__device__ __forceinline__ unsigned rgb_to_gray(unsigned r, unsigned g, unsigned b) {
    int y = (int)((13933u * r + 46871u * g + 4732u * b + 32768u) >> 16);
    return (unsigned)min(max(y, 0), 255);
}

// 4 consecutive pixels as CH 32-bit words (the image base is 4-byte aligned and 4 pixels are 4*CH bytes), unpacked to bytes
template <int CH>
__device__ __forceinline__ void load_group(const uint8_t* __restrict__ img, size_t group, uint8_t (&b)[4 * CH]) {
    if (((uintptr_t)img & 3u) == 0) {   // (uniform) always true for whole images; a row-offset view of Rgb pixels may not be
        const uint32_t* w = reinterpret_cast<const uint32_t*>(img) + group * CH;
#pragma unroll
        for (int i = 0; i < CH; ++i) {
            const uint32_t v = __ldg(w + i);
            b[4 * i] = (uint8_t)v; b[4 * i + 1] = (uint8_t)(v >> 8); b[4 * i + 2] = (uint8_t)(v >> 16); b[4 * i + 3] = (uint8_t)(v >> 24);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4 * CH; ++i) b[i] = img[group * (4 * CH) + i];
    }
}
template <int CH>
__device__ __forceinline__ void store_group(uint8_t* __restrict__ img, size_t group, const uint8_t (&b)[4 * CH]) {
    if (((uintptr_t)img & 3u) == 0) {
        uint32_t* w = reinterpret_cast<uint32_t*>(img) + group * CH;
#pragma unroll
        for (int i = 0; i < CH; ++i)
            w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
    } else {
#pragma unroll
        for (int i = 0; i < 4 * CH; ++i) img[group * (4 * CH) + i] = b[i];
    }
}

struct MapParams;
// What the last block of the statistics kernel does when `update` is queued (fdm.zig:174-254): combine the moments across
// ranks (sharded images), solve the 3x3 problem, leave the map parameters for the map kernel.
struct SolveTail {
    int enabled;
    int pixfmt;
    unsigned int* ticket;      // blocks that have added their partial sums
    unsigned long long* partials;   // [gridDim.x][11]: one slot per block (11 same-line u64 atomics per block from ~1200 blocks
                                    // serialise in one L2 slice: measured ~25 us for a 7 us read; slots + one ticket do not)
    MapParams* out;
    int* status;
    FdmTarget target;
    zb::ShardAll all;          // world == 1: single GPU
};
__device__ void moments_tail(const unsigned long long (*red)[11], const SolveTail& tail);

// sums: {n, Sr, Sg, Sb, Srr, Srg, Srb, Sgg, Sgb, Sbb, non_gray}
template <int CH>
__global__ void __launch_bounds__(256) moments_kernel(const uint8_t* __restrict__ img, size_t n_px, int as_luma,
                                                      unsigned long long* __restrict__ sums, const SolveTail tail) {
    unsigned long long acc[11];
#pragma unroll
    for (int i = 0; i < 11; ++i) acc[i] = 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t n_groups = n_px / 4;   // whole 4-pixel groups; the tail (< 4 pixels) is taken by one thread below
    auto add_px = [&](unsigned (&a)[11], unsigned r, unsigned g, unsigned b) {
        if (CH != 1 && (r != g || g != b)) a[10] += 1;
        if (CH != 1 && as_luma) r = g = b = rgb_to_gray(r, g, b);
        a[0] += 1;
        a[1] += r; a[2] += g; a[3] += b;
        a[4] += r * r; a[5] += r * g; a[6] += r * b;
        a[7] += g * g; a[8] += g * b; a[9] += b * b;
    };
    size_t tail_start = n_groups * 4;   // first pixel the scalar tail below has to take
    if (!as_luma && ((uintptr_t)img & 15u) == 0) {
        // packed path: 16 pixels per iteration as CH 128-bit loads; the 4 pixels of a group are transposed into one word per
        // channel (byte permutes) and every moment of the group is one dot product (dp4a): 6 PRMT + 9 DP4A for 4 pixels
        // instead of ~40 scalar operations per pixel
        unsigned a[11];
#pragma unroll
        for (int i = 0; i < 11; ++i) a[i] = 0;
        int pending = 0;
        const size_t n16 = n_px / 16;
        tail_start = n16 * 16;
#pragma unroll 2
        for (size_t sg = (size_t)blockIdx.x * blockDim.x + threadIdx.x; sg < n16; sg += stride) {
            const uint4* q4 = reinterpret_cast<const uint4*>(img) + sg * CH;
            uint32_t w[4 * CH];
#pragma unroll
            for (int i = 0; i < CH; ++i) {
                const uint4 v = __ldg(q4 + i);
                w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
            }
#pragma unroll
            for (int g4 = 0; g4 < 4; ++g4) {
                const uint32_t* wd = w + g4 * CH;
                uint32_t R, G, B;
                if constexpr (CH == 1) {
                    R = G = B = wd[0];
                } else if constexpr (CH == 3) {
                    const uint32_t w0 = wd[0], w1 = wd[1], w2 = wd[2];                       // r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
                    R = __byte_perm(__byte_perm(w0, w1, 0x0630), w2, 0x5210);              // r0 r1 r2 . -> r0 r1 r2 r3
                    G = __byte_perm(__byte_perm(w0, w1, 0x0741), w2, 0x6210);              // g0 g1 g2 g3
                    B = __byte_perm(__byte_perm(w0, w1, 0x0052), w2, 0x7410);              // b0 b1 . . -> b0 b1 b2 b3
                } else {
                    const uint32_t rg01 = __byte_perm(wd[0], wd[1], 0x5140), rg23 = __byte_perm(wd[2], wd[3], 0x5140);   // r0 r1 g0 g1 | r2 r3 g2 g3
                    R = __byte_perm(rg01, rg23, 0x5410);
                    G = __byte_perm(rg01, rg23, 0x7632);
                    B = __byte_perm(__byte_perm(wd[0], wd[1], 0x0062), __byte_perm(wd[2], wd[3], 0x0062), 0x5410);
                }
                a[0] += 4;
                a[1] = __dp4a(R, 0x01010101u, a[1]); a[2] = __dp4a(G, 0x01010101u, a[2]); a[3] = __dp4a(B, 0x01010101u, a[3]);
                a[4] = __dp4a(R, R, a[4]); a[5] = __dp4a(R, G, a[5]); a[6] = __dp4a(R, B, a[6]);
                a[7] = __dp4a(G, G, a[7]); a[8] = __dp4a(G, B, a[8]); a[9] = __dp4a(B, B, a[9]);
                if (CH != 1) a[10] = __dp4a(__vsetne4((R ^ G) | (G ^ B), 0u), 0x01010101u, a[10]);   // pixels with r != g or g != b
            }
            if (++pending == 1024) {   // 16384 pixels: 16384 * 255^2 < 2^32, flush before the u32 sums can wrap
#pragma unroll
                for (int i = 0; i < 11; ++i) { acc[i] += a[i]; a[i] = 0; }
                pending = 0;
            }
        }
#pragma unroll
        for (int i = 0; i < 11; ++i) acc[i] += a[i];
    } else
    for (size_t base = (size_t)blockIdx.x * blockDim.x + threadIdx.x; base < n_groups; base += stride * 4) {
        unsigned a[11];  // 16 pixels: sums of products <= 16*255^2 fit easily in u32
#pragma unroll
        for (int i = 0; i < 11; ++i) a[i] = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const size_t grp = base + (size_t)j * stride;
            if (grp >= n_groups) break;
            uint8_t b[4 * CH];
            load_group<CH>(img, grp, b);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if constexpr (CH == 1) add_px(a, b[q], b[q], b[q]);
                else add_px(a, b[q * CH], b[q * CH + 1], b[q * CH + 2]);
            }
        }
#pragma unroll
        for (int i = 0; i < 11; ++i) acc[i] += a[i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        unsigned a[11];
#pragma unroll
        for (int i = 0; i < 11; ++i) a[i] = 0;
        for (size_t px = tail_start; px < n_px; ++px) {   // at most 15 pixels
            if constexpr (CH == 1) add_px(a, img[px], img[px], img[px]);
            else add_px(a, img[px * CH], img[px * CH + 1], img[px * CH + 2]);
        }
#pragma unroll
        for (int i = 0; i < 11; ++i) acc[i] += a[i];
    }
    __shared__ unsigned long long sh[8][11];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 11; ++i) {
        unsigned long long v = acc[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) sh[warp][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < 11) {
        unsigned long long v = 0;
        for (int w = 0; w < 8; ++w) v += sh[w][threadIdx.x];
        if (tail.enabled) tail.partials[(size_t)blockIdx.x * 11 + threadIdx.x] = v;
        else atomicAdd(&sums[threadIdx.x], v);
    }
    if (tail.enabled) {
        __shared__ int is_last;
        __shared__ unsigned long long red[16][11];
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            is_last = atomicAdd(tail.ticket, 1u) == gridDim.x - 1u;
        }
        __syncthreads();
        if (is_last) {   // the whole block adds up the slots (16 groups x 11 moments), its first warp finishes the statistics
            __threadfence();
            const unsigned grp = threadIdx.x >> 4, mi = threadIdx.x & 15u;
            if (mi < 11) {
                unsigned long long v = 0;
                for (unsigned b = grp; b < gridDim.x; b += 16) v += __ldcg(&tail.partials[(size_t)b * 11 + mi]);
                red[grp][mi] = v;
            }
            __syncthreads();
            if (threadIdx.x < 32) moments_tail(red, tail);
        }
    }
}

struct MapParams {
    float wf[9], wa[9], bf[3], ba[3];   // f32 fast path of the colour map: weights, (unused), 255*bias, safe distance from k + 1/2 per channel
    double w[9];
    double bias[3];
    double scale, offset;  // gray branch
    int mode;              // 0 colour (fdm.zig:257-271), 1 scalar on u8 (:185-189), 2 gray target on colour source (:191-197)
};

// round(255 * clamp(res, 0, 1)) (fdm.zig:262-270).  255 * clamp(res) and 255 * res agree wherever the clamp is idle, and outside
// it both round to something the integer clamp maps to the same 0 / 255; round-half-away of x is trunc(x) + (x - trunc(x) >= 1/2)
// for x >= 0 and anything <= 0 for x < 0.
__device__ __forceinline__ uint8_t quantize01(double res) {
    const double x = 255.0 * res;
    const int t = __double2int_rz(x);               // saturates far outside the range
    const int r = t + ((x - (double)t) >= 0.5 ? 1 : 0);
    return (uint8_t)min(max(r, 0), 255);
}

// fdm.zig:257-271 for one output channel: f64, the reference's operation order.  Out of line on purpose: it runs for a few values
// in 10^4 and must not be speculated into the fast path.
__device__ __noinline__ uint8_t fdm_exact_channel(int r, int g, int b, int j, const MapParams* __restrict__ p) {
    const double rr = (double)r / 255.0, gg = (double)g / 255.0, bb = (double)b / 255.0;
    return quantize01(rr * p->w[j] + gg * p->w[3 + j] + bb * p->w[6 + j] + p->bias[j]);
}

// The colour map (fdm.zig:257-271) for one pixel: three outputs x_j = 255 * (r/255 * w0j + g/255 * w1j + b/255 * w2j + bias_j),
// rounded half away from zero and clamped.
//
// FP64 is the scarce resource (64 lanes/clk/SM): the reference's 9 multiplies, 9 adds, 3 divisions and 3 roundings per pixel in
// f64 bound the kernel at ~5x the memory time.  So every output is first evaluated in f32 (three FMAs on weights rounded to f32)
// together with a RIGOROUS bound on |x32 - x64|: each of the 3 FMA roundings and each of the 4 rounded constants contributes at
// most 2^-24 of M_j = 255 (|w0j| + |w1j| + |w2j|) + |255 bias_j|, so |x32 - x64| <= 7 * 2^-24 * M_j; the solve stores the
// per-channel constant safe_j = 1/2 - 8 * 2^-24 * M_j.  When x32 is closer than safe_j to its nearest integer, x64 rounds to that
// same integer and the f32 result IS the reference's.  Otherwise (a few values in 10^4) the pixel is recomputed with the
// reference's exact f64 sequence, out of line.  No integer<->float conversion instructions (a quarter-rate pipe): bytes enter
// through the 2^23 exponent trick (PRMT + FADD), x32 is rounded to the nearest integer by adding 1.5 * 2^23, and the result byte is
// the low byte of that sum.  Gray maps are 256-entry byte tables built with the same f64 sequence.
struct MapRegs {
    float w[9], b[3], safe[3];
};
__device__ __forceinline__ float byte_to_float(uint32_t word, int k) {   // byte k of `word` as a float, exactly
    const uint32_t sel = 0x7440u | (uint32_t)k;
    return __uint_as_float(__byte_perm(word, 0x4B000000u, sel)) - 8388608.0f;
}
// returns the packed result bytes (r | g << 8 | b << 16) and sets `bad` when a channel sits too close to a rounding boundary
__device__ __forceinline__ uint32_t map_colour(float rf, float gf, float bf, const MapRegs& m, bool& bad) {
    uint32_t out = 0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float x = fmaf(bf, m.w[6 + j], fmaf(gf, m.w[3 + j], fmaf(rf, m.w[j], m.b[j])));   // ~ 255 * res
        const float t = __fadd_rn(x, 12582912.0f);           // round to the nearest integer (ties are inside the unsafe band)
        const float n = __fsub_rn(t, 12582912.0f);
        const float d = __fsub_rn(x, n);
        bad |= !(fabsf(d) < m.safe[j]);
        // t = 1.5 * 2^23 + round(x): the integer sits in the mantissa, so clamp(round(x), 0, 255) is one subtraction and one
        // min-with-relu (an |x| beyond 2^22 breaks this reading of t, but then d is huge and the pixel is recomputed exactly)
        out |= (uint32_t)__vimin_s32_relu(__float_as_int(t) - 0x4B400000, 255) << (8 * j);
    }
    return out;
}

// A thread maps 16 consecutive pixels when the image is 16-byte aligned (CH 128-bit loads and stores), else 4.
template <int CH>
__global__ void __launch_bounds__(256) fdm_map_kernel(uint8_t* __restrict__ img, size_t n_px, const MapParams* __restrict__ pp) {
    __shared__ uint8_t gray_lut[256];
    __shared__ MapParams sp;   // one copy per block instead of ~30 global loads per thread
    if (threadIdx.x < sizeof(MapParams) / 4) reinterpret_cast<uint32_t*>(&sp)[threadIdx.x] = reinterpret_cast<const uint32_t*>(pp)[threadIdx.x];
    __syncthreads();
    const MapParams& p = sp;
    const int mode = CH == 1 ? 1 : p.mode;
    if (mode != 0) {
        gray_lut[threadIdx.x] = quantize01(((double)threadIdx.x / 255.0) * p.scale + p.offset);
        __syncthreads();
    }
    MapRegs m;
#pragma unroll
    for (int i = 0; i < 9; ++i) m.w[i] = p.wf[i];
#pragma unroll
    for (int j = 0; j < 3; ++j) { m.b[j] = p.bf[j]; m.safe[j] = p.ba[j]; }

    // maps the pixel whose channel bytes are r, g, b (positions inside `q`: byte offsets), in place in the byte array
    auto map_px = [&](uint8_t* q) {
        if constexpr (CH == 1) {
            q[0] = gray_lut[q[0]];
        } else {
            if (mode == 2) {
                const uint8_t res = gray_lut[rgb_to_gray(q[0], q[1], q[2])];
                q[0] = res; q[1] = res; q[2] = res;
                if (CH == 4) q[3] = 0;  // `.{ .r, .g, .b }`: alpha takes its default 0 (color.zig:405, fdm.zig:196)
                return;
            }
            const uint32_t word = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16);
            bool bad = false;
            const uint32_t o = map_colour(byte_to_float(word, 0), byte_to_float(word, 1), byte_to_float(word, 2), m, bad);
            if (bad) {   // exact f64 recomputation of the whole pixel (all three channels read the ORIGINAL r, g, b)
                const int r = q[0], g = q[1], b = q[2];
                q[0] = fdm_exact_channel(r, g, b, 0, pp);
                q[1] = fdm_exact_channel(r, g, b, 1, pp);
                q[2] = fdm_exact_channel(r, g, b, 2, pp);
            } else {
                q[0] = (uint8_t)o; q[1] = (uint8_t)(o >> 8); q[2] = (uint8_t)(o >> 16);
            }
        }
    };
    const size_t tid0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (((uintptr_t)img & 15u) == 0) {
        // grid-stride: a few resident CTAs per SM walk the image (one CTA per 4096 pixels spent a third of its life being launched)
        const size_t n16 = n_px / 16, n_threads = (size_t)gridDim.x * blockDim.x;
        for (size_t tid = tid0; tid <= n16; tid += n_threads)
        if (tid < n16) {
            uint4* q4 = reinterpret_cast<uint4*>(img) + tid * CH;
            uint32_t w[4 * CH];
#pragma unroll
            for (int i = 0; i < CH; ++i) {
                const uint4 v = q4[i];
                w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
            }
            if (CH != 1 && mode == 0) {
                // colour map on packed words: pixel k's bytes sit at byte offset k * CH of the 16 * CH-byte run
                unsigned redo = 0;
                uint32_t res[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    const int o = k * CH;                               // byte offset of r
                    const uint32_t lo = w[o >> 2], hi = w[((o + 3) >> 2) < 4 * CH ? ((o + 3) >> 2) : (4 * CH - 1)];
                    const uint32_t word = __funnelshift_r(lo, hi, (o & 3) * 8);   // r, g, b (, a) in bytes 0..2 (3)
                    bool bad = false;
                    res[k] = map_colour(byte_to_float(word, 0), byte_to_float(word, 1), byte_to_float(word, 2), m, bad);
                    if (bad) {
                        redo |= 1u << k;
                        res[k] = word;                                          // keep the source bytes for the exact pass
                    } else if (CH == 4) {
                        res[k] |= word & 0xFF000000u;                           // alpha is untouched (fdm.zig:268-270)
                    }
                }
                if (redo) {
#pragma unroll
                    for (int k = 0; k < 16; ++k)
                        if (redo & (1u << k)) {
                            const int r = res[k] & 0xFF, g = (res[k] >> 8) & 0xFF, b = (res[k] >> 16) & 0xFF;
                            res[k] = (res[k] & 0xFF000000u) | (uint32_t)fdm_exact_channel(r, g, b, 0, pp) | ((uint32_t)fdm_exact_channel(r, g, b, 1, pp) << 8) |
                                     ((uint32_t)fdm_exact_channel(r, g, b, 2, pp) << 16);
                        }
                }
                if constexpr (CH == 4) {
#pragma unroll
                    for (int k = 0; k < 16; ++k) w[k] = res[k];
                } else {
                    // 16 x 3 bytes -> 12 words: word i holds bytes [4i, 4i + 4) of the stream r0 g0 b0 r1 ...
#pragma unroll
                    for (int i = 0; i < 12; ++i) {
                        const int b0 = 4 * i;                                   // stream byte of the word's byte 0
                        const int k0 = b0 / 3, off = b0 - 3 * k0;              // pixel and channel it starts in
                        // bytes of pixel k0 from channel `off`, then pixel k0 + 1 (and k0 + 2 when off == 2 ... covered by 3 pixels)
                        const uint32_t a = res[k0] >> (8 * off);                // (3 - off) valid bytes
                        const uint32_t b = k0 + 1 < 16 ? res[k0 + 1] : 0u;      // 3 valid bytes
                        const uint32_t c = k0 + 2 < 16 ? res[k0 + 2] : 0u;
                        uint32_t v;
                        if (off == 0) v = (a & 0x00FFFFFFu) | (b << 24);
                        else if (off == 1) v = (a & 0x0000FFFFu) | ((b & 0x0000FFFFu) << 16);
                        else v = (a & 0x000000FFu) | ((b & 0x00FFFFFFu) << 8);
                        (void)c;
                        w[i] = v;
                    }
                }
            } else {
                uint8_t* bytes = reinterpret_cast<uint8_t*>(w);
#pragma unroll
                for (int k = 0; k < 16; ++k) map_px(bytes + k * CH);
            }
#pragma unroll
            for (int i = 0; i < CH; ++i) q4[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
        } else {   // tid == n16: the tail (< 16 pixels), byte by byte
            for (size_t px = n16 * 16; px < n_px; ++px) map_px(img + px * CH);
        }
        return;
    }
    const size_t tid = tid0;
    const size_t n_groups = n_px / 4;
    if (tid < n_groups) {
        uint8_t b[4 * CH];
        load_group<CH>(img, tid, b);
#pragma unroll
        for (int q = 0; q < 4; ++q) map_px(b + q * CH);
        store_group<CH>(img, tid, b);
    } else if (tid == n_groups) {   // the tail (< 4 pixels), byte by byte
        for (size_t px = n_groups * 4; px < n_px; ++px) map_px(img + px * CH);
    }
}

static SolveTail no_tail() {
    SolveTail t;
    memset(&t, 0, sizeof(t));
    return t;
}

int moments_device(const zb_image* img, int pixfmt, int as_luma, uint64_t* sums11, cudaStream_t s) {
    if (!img || !sums11) return ZB_ERR_INVALID_ARGUMENT;
    if (pixfmt != ZB_PIX_U8 && pixfmt != ZB_PIX_RGB8 && pixfmt != ZB_PIX_RGBA8) return ZB_ERR_UNSUPPORTED;  // fdm.zig:20
    if (img->stride != img->cols) return ZB_ERR_UNSUPPORTED;  // the reference walks image.data linearly (fdm.zig:82)
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const size_t n_px = (size_t)img->rows * img->cols;
    Scratch d;
    if ((rc = d.alloc(11 * sizeof(uint64_t), s))) return rc;
    ZB_CUDA(cudaMemsetAsync(d.p, 0, 11 * sizeof(uint64_t), s));
    if (n_px > 0) {
        const unsigned blocks = (unsigned)std::min<size_t>((size_t)di.sm_count * 8, (n_px + 255) / 256);
        const uint8_t* p = (const uint8_t*)img->data;
        auto* ds = d.as<unsigned long long>();
        switch (pixfmt) {
            case ZB_PIX_U8: moments_kernel<1><<<blocks, 256, 0, s>>>(p, n_px, as_luma, ds, no_tail()); break;
            case ZB_PIX_RGB8: moments_kernel<3><<<blocks, 256, 0, s>>>(p, n_px, as_luma, ds, no_tail()); break;
            default: moments_kernel<4><<<blocks, 256, 0, s>>>(p, n_px, as_luma, ds, no_tail()); break;
        }
        ZB_LAUNCHED();
    }
    ZB_CUDA(cudaMemcpyAsync(sums11, d.p, 11 * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    return ZB_OK;
}

// mean (stats.zig:283-286) and unbiased covariance (:301-320) of x/255 from the integer moments
ZB_HD inline double i128_to_double(__int128 v) {   // two roundings at most 2^-53 relative each; no library call on the device
    const bool neg = v < 0;
    const unsigned __int128 a = neg ? (unsigned __int128)(-v) : (unsigned __int128)v;
    const double d = (double)(unsigned long long)(a >> 64) * 18446744073709551616.0 + (double)(unsigned long long)a;
    return neg ? -d : d;
}
ZB_HD inline void stats_from_moments(const unsigned long long* m, double mean[3], double cov[9]) {
    const double n = (double)m[0];
    for (int i = 0; i < 3; ++i) mean[i] = m[0] ? ((double)m[1 + i] / n) / 255.0 : 0.0;
    for (int i = 0; i < 9; ++i) cov[i] = 0.0;
    if (m[0] <= 1) return;
    const int idx[3][3] = {{4, 5, 6}, {5, 7, 8}, {6, 8, 9}};
    const double denom = i128_to_double((__int128)m[0] * (__int128)(m[0] - 1) * 65025);
    for (int i = 0; i < 3; ++i)
        for (int j = i; j < 3; ++j) {
            const __int128 num = (__int128)m[0] * (__int128)m[idx[i][j]] - (__int128)m[1 + i] * (__int128)m[1 + j];
            const double c = i128_to_double(num) / denom;
            cov[i * 3 + j] = c;
            cov[j * 3 + i] = c;
        }
}

// scalar 3x3 product in the reference's gemm order (Matrix.zig:806-817: 27 ops < 512 -> scalar path)
ZB_HD inline void matmul3(const double* a, const double* b, double* out) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double acc = 0;
            for (int k = 0; k < 3; ++k) acc += a[i * 3 + k] * b[k * 3 + j];
            out[i * 3 + j] = 0.0 + 1.0 * acc;
        }
}

// fdm.zig:174-254: the map parameters from the source moments and the target statistics
ZB_HD inline int fdm_solve(const unsigned long long* m, const FdmTarget& t, int pixfmt, MapParams& p) {
    double source_mean[3], scov[9];
    stats_from_moments(m, source_mean, scov);
    for (int i = 0; i < 9; ++i) p.w[i] = 0;
    for (int i = 0; i < 3; ++i) p.bias[i] = 0;
    p.scale = 1.0;
    p.offset = 0.0;
    if (pixfmt == ZB_PIX_U8 || t.is_gray) {  // :177-198
        const double source_var = scov[0];
        p.scale = source_var > 1e-10 ? sqrt(t.s[0] / source_var) : 1.0;
        p.offset = t.mean[0] - source_mean[0] * p.scale;
        p.mode = pixfmt == ZB_PIX_U8 ? 1 : 2;
        return ZB_OK;
    }
    double us[9], ss[3], v[9], e[3];   // :199-254
    if (svd_gr_core<double>(scov, 3, 3, ZB_SVD_SKINNY_U, false, us, 3, ss, v, e) != 0) return ZB_ERR_NOT_CONVERGED;
    double sigma[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 3; ++i)
        if (ss[i] > 1e-10) sigma[i * 3 + i] = sqrt(t.s[i] / ss[i]);
    double ut_t[9], w_temp[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) ut_t[i * 3 + j] = t.u[j * 3 + i];
    matmul3(us, sigma, w_temp);
    matmul3(w_temp, ut_t, p.w);
    for (int j = 0; j < 3; ++j) {
        double sum = 0;
        for (int k = 0; k < 3; ++k) sum += source_mean[k] * p.w[k * 3 + j];
        p.bias[j] = t.mean[j] - sum;
    }
    p.mode = 0;
    return ZB_OK;
}

// the f32 constants of the map's fast path (see map_colour)
ZB_HD inline void finish_map_params(MapParams& p) {
    for (int i = 0; i < 9; ++i) { p.wf[i] = (float)p.w[i]; p.wa[i] = 0.0f; }
    for (int j = 0; j < 3; ++j) {
        p.bf[j] = (float)(255.0 * p.bias[j]);
        const double M = 255.0 * (fabs(p.w[j]) + fabs(p.w[3 + j]) + fabs(p.w[6 + j])) + fabs(255.0 * p.bias[j]);
        const double safe = 0.5 - 8.0 * 5.9604644775390625e-08 * M - 1e-6;   // 8 * 2^-24 * M, and x must stay below 2^22 for the rounding trick
        p.ba[j] = (safe > 0.0 && M < 4.0e6) ? (float)safe : -1.0f;           // -1: every pixel takes the exact path
    }
}

__global__ void fdm_solve_kernel(const unsigned long long* __restrict__ m, FdmTarget t, int pixfmt, MapParams* __restrict__ out,
                                 int* __restrict__ status) {
    MapParams p;
    const int rc = fdm_solve(m, t, pixfmt, p);
    finish_map_params(p);
    *out = p;
    *status = rc;
}

// Runs in the first warp of the last block of moments_kernel.  Sharded images: every rank stores its 11 sums into its slot of
// every rank's control block (plain peer stores over NVLink, then one release flag per rank), waits for the other ranks' flags
// and adds the slots in rank order -- an 88-byte all-gather that costs one NVLink round trip instead of a collective launch.
__device__ void moments_tail(const unsigned long long (*red)[11], const SolveTail& tail) {
    __shared__ unsigned long long m[11];
    const int lane = threadIdx.x;
    if (lane < 11) {
        unsigned long long v = 0;
        for (int g = 0; g < 16; ++g) v += red[g][lane];   // integer sums: any order gives the same bits
        m[lane] = v;
    }
    __syncwarp();
    const zb::ShardAll& a = tail.all;
    if (a.world > 1) {
        const int par = (int)(a.epoch & 1ull);
        if (lane < 11)
            for (int r = 0; r < a.world; ++r) a.ctrl[r]->gather[par][a.rank][lane] = m[lane];
        __threadfence_system();
        __syncwarp();
        if (lane < a.world) st_release_sys(&a.ctrl[lane]->gather[par][a.rank][15], a.epoch);
        zb::ShardCtrl* me = a.ctrl[a.rank];
        if (lane < a.world) zb::shard_wait_ge(&me->gather[par][lane][15], a.epoch, me);
        __syncwarp();
        if (lane < 11) {
            unsigned long long v = 0;
            for (int r = 0; r < a.world; ++r) v += *(volatile unsigned long long*)&me->gather[par][r][lane];
            m[lane] = v;
        }
        __syncwarp();
    }
    if (lane == 0) {
        *tail.ticket = 0;
        MapParams p;
        const int rc = fdm_solve(m, tail.target, tail.pixfmt, p);
        finish_map_params(p);
        *tail.out = p;
        *tail.status = rc;
    }
}

// the target's 3x3 decomposition on the host: the same fixed-size routine the device solve uses
static uint64_t svd3_host(const double* cov, double* u, double* q, double* v) {
    double e[3] = {0, 0, 0};
    return svd_gr_core<double>(cov, 3, 3, ZB_SVD_SKINNY_U, false, u, 3, q, v, e);
}

// fdm.zig:92-121
int set_target_from_moments(zb_fdm* f, const uint64_t* m) {
    double cov[9];
    stats_from_moments((const unsigned long long*)m, f->target_mean, cov);
    f->target_is_gray = (f->pixfmt == ZB_PIX_U8) || (m[10] == 0);
    memset(f->target_u, 0, sizeof(f->target_u));
    f->target_s[0] = f->target_s[1] = f->target_s[2] = 0;
    if (f->target_is_gray) {
        f->target_s[0] = cov[0];
    } else {
        double v[9];
        if (svd3_host(cov, f->target_u, f->target_s, v) != 0) return ZB_ERR_NOT_CONVERGED;
    }
    f->has_target = true;
    return ZB_OK;
}

constexpr unsigned kMaxMomentBlocks = 2048;

// The zeroing is queued on `s`, the stream of the first moments pass: the fused solve tail reads the block ticket (word 11 of d_m),
// so the memset must be ordered before that kernel on its own stream, not on the legacy NULL stream.
int ensure_device_state(zb_fdm* f, cudaStream_t s) {
    if (f->d_m) return ZB_OK;
    ZB_CUDA(cudaMalloc(&f->d_m, (12 + (size_t)kMaxMomentBlocks * 11) * sizeof(unsigned long long)));   // 11 sums, the block ticket, per-block slots
    ZB_CUDA(cudaMalloc(&f->d_params, sizeof(MapParams)));
    ZB_CUDA(cudaMalloc(&f->d_status, sizeof(int)));
    ZB_CUDA(cudaMemsetAsync(f->d_m, 0, 12 * sizeof(unsigned long long), s));
    ZB_CUDA(cudaMemsetAsync(f->d_status, 0, sizeof(int), s));
    return ZB_OK;
}

FdmTarget target_of(const zb_fdm* f) {
    FdmTarget t;
    memcpy(t.mean, f->target_mean, sizeof(t.mean));
    memcpy(t.u, f->target_u, sizeof(t.u));
    memcpy(t.s, f->target_s, sizeof(t.s));
    t.is_gray = f->target_is_gray ? 1 : 0;
    return t;
}

// Queue the moment pass of `img` into f->d_m (no host synchronisation).  With `solve` the last block of the kernel also finishes
// the statistics (all-gather across ranks when `all` has more than one), solves the 3x3 problem and writes the map parameters:
// the separate one-thread solve launch and the memset node are gone.  f->d_m is zero on entry and on exit in that mode.
int moments_enqueue(zb_fdm* f, const zb_image* img, int as_luma, cudaStream_t s, bool solve, const ShardAll* all) {
    if (img->stride != img->cols) return ZB_ERR_UNSUPPORTED;  // the reference walks image.data linearly (fdm.zig:82)
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if ((rc = ensure_device_state(f, s))) return rc;
    const size_t n_px = (size_t)img->rows * img->cols;
    SolveTail tail = no_tail();
    if (solve) {
        tail.enabled = 1;
        tail.pixfmt = f->pixfmt;
        tail.ticket = reinterpret_cast<unsigned int*>(f->d_m + 11);
        tail.partials = f->d_m + 12;
        tail.out = (MapParams*)f->d_params;
        tail.status = f->d_status;
        tail.target = target_of(f);
        if (all) tail.all = *all;
        else { tail.all.world = 1; tail.all.rank = 0; }
    } else {
        ZB_CUDA(cudaMemsetAsync(f->d_m, 0, 11 * sizeof(unsigned long long), s));
    }
    if (n_px > 0 || solve) {
        const unsigned blocks = (unsigned)std::max<size_t>(1, std::min<size_t>(std::min<size_t>((size_t)di.sm_count * 8, kMaxMomentBlocks), (n_px + 255) / 256));
        const uint8_t* p = (const uint8_t*)img->data;
        switch (f->pixfmt) {
            case ZB_PIX_U8: moments_kernel<1><<<blocks, 256, 0, s>>>(p, n_px, as_luma, f->d_m, tail); break;
            case ZB_PIX_RGB8: moments_kernel<3><<<blocks, 256, 0, s>>>(p, n_px, as_luma, f->d_m, tail); break;
            default: moments_kernel<4><<<blocks, 256, 0, s>>>(p, n_px, as_luma, f->d_m, tail); break;
        }
        ZB_LAUNCHED();
    }
    return ZB_OK;
}

int map_enqueue(zb_fdm* f, cudaStream_t s) {
    const size_t n_px = (size_t)f->source.rows * f->source.cols;
    if (n_px == 0) return ZB_OK;
    MapParams* dp = (MapParams*)f->d_params;
    uint8_t* img = (uint8_t*)f->source.data;
    // one thread per 16-pixel run (16-byte aligned images) or 4-pixel group, one more for the tail
    unsigned blocks = (((uintptr_t)img) & 15u) == 0 ? div_up(n_px / 16 + 1, 256) : div_up(n_px / 4 + 1, 256);
    if ((((uintptr_t)img) & 15u) == 0) {   // the aligned path strides over the image: 8 CTAs per SM are plenty
        DeviceInfo di;
        if (device_info(&di) == ZB_OK && blocks > 8u * (unsigned)di.sm_count) blocks = 8u * (unsigned)di.sm_count;
    }
    switch (channels_of(f->pixfmt)) {
        case 1: fdm_map_kernel<1><<<blocks, 256, 0, s>>>(img, n_px, dp); break;
        case 3: fdm_map_kernel<3><<<blocks, 256, 0, s>>>(img, n_px, dp); break;
        default: fdm_map_kernel<4><<<blocks, 256, 0, s>>>(img, n_px, dp); break;
    }
    ZB_LAUNCHED();
    t_last_kernel = "fdm_map";
    return ZB_OK;
}

// fdm.zig:174-272 with the source moments already in f->d_m: solve on the device (one thread), then map -- all queued on `s`
int solve_and_map(zb_fdm* f, cudaStream_t s) {
    const size_t n_px = (size_t)f->source.rows * f->source.cols;
    if (n_px == 0) return ZB_OK;
    fdm_solve_kernel<<<1, 1, 0, s>>>(f->d_m, target_of(f), f->pixfmt, (MapParams*)f->d_params, f->d_status);
    ZB_LAUNCHED();
    ZB_CUDA(cudaMemsetAsync(f->d_m, 0, 11 * sizeof(unsigned long long), s));   // the fused-tail mode expects zeroed sums
    return map_enqueue(f, s);
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" {

int zb_fdm_create(zb_fdm** out, int pixfmt) {
    if (!out) return ZB_ERR_INVALID_ARGUMENT;
    if (pixfmt != ZB_PIX_U8 && pixfmt != ZB_PIX_RGB8 && pixfmt != ZB_PIX_RGBA8) return ZB_ERR_UNSUPPORTED;  // fdm.zig:20
    zb_fdm* f = new zb_fdm();
    memset(f, 0, sizeof(*f));
    f->pixfmt = pixfmt;
    *out = f;
    return ZB_OK;
}
int zb_fdm_destroy(zb_fdm* f) {
    if (f) {
        if (f->d_m) cudaFree(f->d_m);
        if (f->d_params) cudaFree(f->d_params);
        if (f->d_status) cudaFree(f->d_status);
    }
    delete f;
    return ZB_OK;
}

int zb_fdm_moments(const zb_image* img, int pixfmt, int as_luma, uint64_t* sums11, zb_stream s) {
    return moments_device(img, pixfmt, as_luma, sums11, (cudaStream_t)s);
}

int zb_fdm_set_target_moments(zb_fdm* f, const uint64_t* sums11) {
    if (!f || !sums11) return ZB_ERR_INVALID_ARGUMENT;
    return set_target_from_moments(f, sums11);
}

int zb_fdm_set_target(zb_fdm* f, const zb_image* target, zb_stream s) {
    if (!f || !target) return ZB_ERR_INVALID_ARGUMENT;
    uint64_t m[11];
    int rc = moments_device(target, f->pixfmt, 0, m, (cudaStream_t)s);
    if (rc) return rc;
    return set_target_from_moments(f, m);
}

int zb_fdm_set_source(zb_fdm* f, zb_image* source) {
    if (!f || !source) return ZB_ERR_INVALID_ARGUMENT;
    if (source->stride != source->cols) return ZB_ERR_UNSUPPORTED;
    f->source = *source;
    f->has_source = true;
    return ZB_OK;
}

int zb_fdm_update_with_moments(zb_fdm* f, const uint64_t* source_sums11, zb_stream s) {
    if (!f || !source_sums11) return ZB_ERR_INVALID_ARGUMENT;
    if (!f->has_target) return ZB_ERR_NO_TARGET_SET;  // fdm.zig:142
    if (!f->has_source) return ZB_ERR_NO_SOURCE_SET;  // fdm.zig:143
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if ((rc = ensure_device_state(f, (cudaStream_t)s))) return rc;
    // (pageable source: the copy is staged before the call returns, so the caller's array may be reused)
    ZB_CUDA(cudaMemcpyAsync(f->d_m, source_sums11, 11 * sizeof(unsigned long long), cudaMemcpyHostToDevice, (cudaStream_t)s));
    return solve_and_map(f, (cudaStream_t)s);
}

int zb_fdm_update(zb_fdm* f, zb_stream s) {
    if (!f) return ZB_ERR_INVALID_ARGUMENT;
    if (!f->has_target) return ZB_ERR_NO_TARGET_SET;
    if (!f->has_source) return ZB_ERR_NO_SOURCE_SET;
    const int as_luma = (f->pixfmt != ZB_PIX_U8 && f->target_is_gray) ? 1 : 0;  // fdm.zig:155-162
    if ((size_t)f->source.rows * f->source.cols == 0) return ZB_OK;
    int rc = moments_enqueue(f, &f->source, as_luma, (cudaStream_t)s, true, nullptr);   // statistics + solve: one kernel
    if (rc) return rc;                                                                   // no device-to-host round trip
    return map_enqueue(f, (cudaStream_t)s);
}

/* ---- sharded image: every rank holds a row block of the source / target (SURVEY 8(e)) ---- */
int zb_shard_fdm_set_target(zb_shard_comm* c, zb_fdm* f, const zb_image* target_block, zb_stream stream) {
    if (!c || !f || !target_block) return ZB_ERR_INVALID_ARGUMENT;
    cudaStream_t s = (cudaStream_t)stream;
    int rc = moments_enqueue(f, target_block, 0, s, false, nullptr);
    if (rc) return rc;
    if ((rc = shard_allreduce(c, f->d_m, 11, 2, s))) return rc;          // exact integer sums: order-independent
    uint64_t m[11];
    ZB_CUDA(cudaMemcpyAsync(m, f->d_m, sizeof(m), cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaMemsetAsync(f->d_m, 0, 11 * sizeof(unsigned long long), s));
    ZB_CUDA(cudaStreamSynchronize(s));
    return set_target_from_moments(f, m);
}

int zb_shard_fdm_update(zb_shard_comm* c, zb_fdm* f, zb_stream stream) {
    if (!c || !f) return ZB_ERR_INVALID_ARGUMENT;
    if (!f->has_target) return ZB_ERR_NO_TARGET_SET;
    if (!f->has_source) return ZB_ERR_NO_SOURCE_SET;
    cudaStream_t s = (cudaStream_t)stream;
    const int as_luma = (f->pixfmt != ZB_PIX_U8 && f->target_is_gray) ? 1 : 0;
    int rc;
    if (shard_world(c) > 1 && !shard_peer_ok(c)) {
        // no peer mappings: NCCL all-reduce of the 11 sums between the statistics kernel and the one-thread solve
        if ((rc = moments_enqueue(f, &f->source, as_luma, s, false, nullptr))) return rc;
        if ((rc = shard_allreduce(c, f->d_m, 11, 2, s))) return rc;
        if ((size_t)f->source.rows * f->source.cols == 0) return ZB_OK;
        return solve_and_map(f, s);
    }
    ShardAll all;
    shard_all(c, true, &all);
    if ((rc = moments_enqueue(f, &f->source, as_luma, s, true, &all))) return rc;
    return map_enqueue(f, s);
}

int zb_fdm_status(zb_fdm* f, zb_stream s) {
    if (!f) return ZB_ERR_INVALID_ARGUMENT;
    if (!f->d_status) return ZB_OK;
    int st = 0;
    ZB_CUDA(cudaMemcpyAsync(&st, f->d_status, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)s));
    ZB_CUDA(cudaStreamSynchronize((cudaStream_t)s));
    return st;
}

int zb_fdm_match(zb_fdm* f, zb_image* source, const zb_image* target, zb_stream s) {  // fdm.zig:133-137
    int rc;
    if ((rc = zb_fdm_set_target(f, target, s))) return rc;
    if ((rc = zb_fdm_set_source(f, source))) return rc;
    return zb_fdm_update(f, s);
}

int zb_host_fdm_match(zb_image* source, const zb_image* target, int pixfmt) {
    if (!source || !target) return ZB_ERR_INVALID_ARGUMENT;
    if (source->stride != source->cols || target->stride != target->cols) return ZB_ERR_UNSUPPORTED;
    zb_fdm* f = nullptr;
    int rc = zb_fdm_create(&f, pixfmt);
    if (rc) return rc;
    HostStage st;  // src slot = target image, dst slot = source image (modified in place)
    const size_t pb = pixel_bytes(pixfmt);
    rc = st.begin(target, source, pixfmt);
    if (!rc) {
        cudaError_t e = cudaMemcpyAsync(st.ddst.data, source->data, (size_t)source->rows * source->cols * pb, cudaMemcpyHostToDevice, st.stream);
        if (e != cudaSuccess) rc = set_cuda_error(e, "upload source", __FILE__, __LINE__);
    }
    if (!rc) rc = zb_fdm_match(f, &st.ddst, &st.dsrc, (zb_stream)st.stream);
    if (!rc) rc = st.finish(source, pixfmt);
    zb_fdm_destroy(f);
    return rc;
}

}  // extern "C"
