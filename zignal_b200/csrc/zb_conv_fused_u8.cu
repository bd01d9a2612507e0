// zb_conv_fused_u8.cu -- single-pass separable convolution of interleaved Rgba(u8) for sm_90a.
//
// Reference semantics (convolution.zig:340-431 -> convolveSeparablePlane(u8, i32), :441-647): Q8 taps
// round(k*256), horizontal pass into an i32 temp (not rounded), vertical pass, one divClampU8(65536)
// at the end.  The reference de-interleaves into planes first; per-channel results are identical, so
// this kernel keeps pixels interleaved: one 32-bit word per pixel in HBM, 4 B in + 4 B out per pixel
// (the reference's data flow moves ~40 B/px: split, i32 temp plane write+read per channel, merge).
//
// Structure = the RGBA f32 kernel (zb_conv_fused.cu): persistent CTAs, (band x 256-px strip)
// work units in band-major order, 8-row chunks landed by TMA (2-D tensor of 32-bit pixels, zero OOB
// fill, 16-px halo each side so every thread's 96-byte window is 16-byte aligned), horizontal pass
// into a 24-row shared ring of per-channel sums, vertical pass from the ring, both register-
// blocked 8 outputs per thread; border pixels patched in the stage per resolveIndex.
//
// One kernel template carries three pipelines for the multiply-adds (Pipe); they share the TMA producer, the unit loop, the
// border fixups and the barriers, and differ only in h_pass / v_pass and in the ring's row size:
//   IMAD  i32 accumulators, the taps as uniform-register operands;
//   FFMA  the same integer sums in f32, exact when the host proves 255 * sum|kx| * sum|ky| <= 2^24 (FFMA has twice the IMAD rate);
//   DP    dp4a / dp2a on byte taps with u16 horizontal sums: half the ring, two CTAs per SM.
// With 120 IMAD/px at 15 taps and only 8 B/px of HBM traffic this kernel is bound by the integer/FMA pipe, not by HBM
// (DESIGN.md 4.1b).
//
// Accumulators are i32: the host proves 255 * sum|kx| * sum|ky| + 32768 < 2^31 (true for any
// normalised kernel); otherwise the generic path (i64 accumulators, saturating i32 temp) is used.
#include "zb_conv.h"
#include "zb_device.cuh"
#include "zb_tma.cuh"

#include <type_traits>

namespace zb {

namespace {

constexpr int TW = 256;
constexpr int CHUNK = 8;
constexpr int PAD = 16;                          // halo pixels each side of the strip in the stage
constexpr int SW = TW + 2 * PAD;                 // stage row: 288 pixels
// TMA boxes are limited to 256 elements per dimension, so a stage is two boxes of 144 pixels x 8 rows side by side:
// stage layout [2 blocks][8 rows][144 px].  144 is a multiple of 4, so a 16-byte chunk never straddles the blocks.
constexpr int BW = SW / 2;                       // 144
constexpr int BLOCK_ROW_BYTES = BW * 4;          // 576
constexpr int BLOCK_BYTES = BLOCK_ROW_BYTES * CHUNK;  // 4608
constexpr int STAGE_BYTES = 2 * BLOCK_BYTES;     // 9216
__device__ __forceinline__ uint32_t stage_px(uint32_t stage, int rr, int xx) {
    const int b = xx >= BW ? 1 : 0;
    return stage + (uint32_t)(b * BLOCK_BYTES + rr * BLOCK_ROW_BYTES + (xx - b * BW) * 4);
}
constexpr int NSTAGE = 3;
constexpr int RING_ROWS = 24;
constexpr int NTHREADS = 256;
constexpr int MAX_HALF = 8;
constexpr int MAXK = 2 * MAX_HALF + 1;

enum class Pipe { IMAD, FFMA, DP };
// A ring row holds the horizontal sums of 256 pixels: int4 / float4 per pixel, or two u16 pairs per pixel for DP.
constexpr int ring_row_bytes(Pipe P) { return P == Pipe::DP ? TW * 8 : TW * 16; }
constexpr int smem_bytes(Pipe P) { return NSTAGE * STAGE_BYTES + RING_ROWS * ring_row_bytes(P) + 64 + 1024; }
constexpr int ctas_per_sm(Pipe P) { return P == Pipe::DP ? 2 : 1; }

// This layout is part of the kernels' speed; time any change to it.  ptxas pairs words at 8-byte aligned addresses into 64-bit
// uniform loads, so moving the DP tables by 4 bytes reschedules the DP kernels.  Moving the scalars by 16 bytes, with the code
// unchanged instruction for instruction, cost 0.1-0.2 % at 8192^2 on an H100 SXM (700 W).
struct U8Params {
    int kx[MAXK];
    int ky[MAXK];
    float kxf[MAXK];  // the same Q8 taps as floats (FFMA pipeline)
    float kyf[MAXK];  // ky_q8 / 65536: the vertical sums come out as acc / 65536 (exact), ready for round_clamp_byte
    const uint32_t* src;
    uint32_t* dst;
    unsigned long long src_pitch_px, dst_pitch_px;
    int rows, cols, border;
    int n_strips, n_bands, band_rows;
    int row0, row1;  // output rows this launch produces
    int fix;  // 1 if out-of-range stage entries need patching (border != zero)
    unsigned kxs[4][5];  // DP pipeline: horizontal taps packed four bytes per word, delayed by sh = 0..3 bytes (tap 4q + b - sh in byte b,
                         // zero beyond the kernel): a window that starts sh bytes into a word meets ALIGNED words with shifted taps
                         // instead of being funnel-shifted into place
    unsigned ky4[5];  // DP pipeline: vertical taps, tap 4q + b in byte b; dp2a.lo reads bytes 0,1 (taps 4q, 4q+1), dp2a.hi bytes 2,3
};

// Work unit u = (band, strip) in band-major order: the strip's first column, its output rows [ra, rb), and the chunks it reads
// (one halo chunk above and one below the band's).
struct Unit {
    int x0, ra, rb, n_in;
};
__device__ __forceinline__ Unit decode_unit(int u, const U8Params& p) {
    const int band = u / p.n_strips, strip = u - band * p.n_strips;
    const int ra = p.row0 + band * p.band_rows;
    const int rb = min(ra + p.band_rows, p.row1);
    return {strip * TW, ra, rb, (rb - ra + CHUNK - 1) / CHUNK + 2};
}

// Patch stage entries whose pixel lies outside the image (TMA wrote zeros there).
__device__ __noinline__ void fixup_stage_u8(uint32_t stage, int y0, int xs0, bool fix_x, bool fix_rows, const U8Params& p) {
    if (fix_x) {
        const int nleft = xs0 < 0 ? min(-xs0, SW) : 0;
        const int r0 = max(0, p.cols - xs0);
        const int r1 = min(SW, p.cols - xs0 + MAX_HALF);
        const int per_row = nleft + max(0, r1 - r0);
        for (int idx = threadIdx.x; idx < CHUNK * per_row; idx += NTHREADS) {
            const int rr = idx / per_row, e = idx - rr * per_row;
            const int xx = e < nleft ? e : r0 + (e - nleft);
            const int y = y0 + rr, x = xs0 + xx;
            if (y < 0 || y >= p.rows) continue;
            const int rx = resolve_index(x, p.cols, p.border);
            uint32_t v = 0;
            if (rx >= 0) {
                const int sx = rx - xs0;
                if (sx >= 0 && sx < SW) v = lds32(stage_px(stage, rr, sx));
                else v = __ldg(p.src + (size_t)y * p.src_pitch_px + rx);
            }
            sts32(stage_px(stage, rr, xx), v);
        }
    }
    if (fix_rows) {
        for (int idx = threadIdx.x; idx < CHUNK * SW; idx += NTHREADS) {
            const int rr = idx / SW, xx = idx - rr * SW;
            const int y = y0 + rr, x = xs0 + xx;
            if (y >= 0 && y < p.rows) continue;
            const int ry = resolve_index(y, p.rows, p.border);
            const int rx = resolve_index(x, p.cols, p.border);
            uint32_t v = 0;
            if (ry >= 0 && rx >= 0) v = __ldg(p.src + (size_t)ry * p.src_pitch_px + rx);
            sts32(stage_px(stage, rr, xx), v);
        }
    }
}

// ---- IMAD and FFMA: one loop nest on int4 or float4 accumulators ----------------------------------------------------------------
// FFMA: when 255 * sum|kx| * sum|ky| <= 2^24 every partial sum is an integer of magnitude <= 2^24, hence exactly representable in
// f32, and an FFMA of exact integers whose result is representable returns it exactly -- so the whole Q8 pipeline can run on the
// (faster) FFMA path with bit-identical results.
template <Pipe P>
using Acc4 = std::conditional_t<P == Pipe::FFMA, float4, int4>;

__device__ __forceinline__ void mac4(int4& acc, const int4& v, int k) {
    acc.x += v.x * k;
    acc.y += v.y * k;
    acc.z += v.z * k;
    acc.w += v.w * k;
}
__device__ __forceinline__ void mac4(float4& acc, const float4& v, float k) {
    acc.x = fmaf(v.x, k, acc.x);
    acc.y = fmaf(v.y, k, acc.y);
    acc.z = fmaf(v.z, k, acc.z);
    acc.w = fmaf(v.w, k, acc.w);
}
// Byte k of `w` as a float without an I2F (the conversion pipe runs at a quarter of the FMA rate and the horizontal pass needs
// ~11 of them per output pixel): PRMT drops the byte into the mantissa of 2^23, one FADD removes the 2^23.  Exact.
__device__ __forceinline__ float byte_f32(uint32_t w, int k) {
    return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440u | (uint32_t)k)) - 8388608.0f;
}
// divClampU8(65536, acc) (convolution.zig:18-22) on u = acc / 65536 held exactly in f32 (the vertical taps carry the 2^-16):
// round half away from zero, clamp to [0, 255], and return the integer in the low byte -- no F2I.  u + 1.5 * 2^23 rounds to the
// nearest integer (ties to even); the one case where that differs from half-away for u >= 0 is u = k + 1/2 with k even.
__device__ __forceinline__ uint32_t round_clamp_byte(float u) {
    const float t = __fadd_rn(u, 12582912.0f);
    float r = __fsub_rn(t, 12582912.0f);
    if (__fsub_rn(u, r) == 0.5f) r = __fadd_rn(r, 1.0f);
    r = fminf(fmaxf(r, 0.0f), 255.0f);
    return __float_as_uint(__fadd_rn(r, 8388608.0f)) & 0xFFu;
}
// divClampU8(65536, acc) for |acc| < 2^31 - 32768 (convolution.zig:18-22)
__device__ __forceinline__ uint32_t div_clamp_65536(int acc) {
    const int t = acc + 32768 + ((acc >> 31) & -65536);  // acc - 32768 when negative
    return t < 0 ? 0u : min((uint32_t)t >> 16, 255u);     // trunc toward zero, then clamp
}
__device__ __forceinline__ uint32_t pack_rgba(const float4& a) {
    return round_clamp_byte(a.x) | (round_clamp_byte(a.y) << 8) | (round_clamp_byte(a.z) << 16) | (round_clamp_byte(a.w) << 24);
}
__device__ __forceinline__ uint32_t pack_rgba(const int4& a) {
    return div_clamp_65536(a.x) | (div_clamp_65536(a.y) << 8) | (div_clamp_65536(a.z) << 16) | (div_clamp_65536(a.w) << 24);
}
template <Pipe P>
__device__ __forceinline__ Acc4<P> unpack_px(uint32_t w) {
    if constexpr (P == Pipe::FFMA) return make_float4(byte_f32(w, 0), byte_f32(w, 1), byte_f32(w, 2), byte_f32(w, 3));
    else return make_int4((int)(w & 0xffu), (int)((w >> 8) & 0xffu), (int)((w >> 16) & 0xffu), (int)(w >> 24));
}
template <Pipe P>
__device__ __forceinline__ Acc4<P> lds_acc(uint32_t addr) {
    if constexpr (P == Pipe::FFMA) return lds128(addr);
    else return lds128_i(addr);
}
template <Pipe P>
__device__ __forceinline__ void sts_acc(uint32_t addr, const Acc4<P>& v) {
    if constexpr (P == Pipe::FFMA) sts128(addr, v);
    else sts128_i(addr, v);
}
template <Pipe P>
__device__ __forceinline__ auto htap(const U8Params& p, int t) {
    if constexpr (P == Pipe::FFMA) return p.kxf[t];
    else return p.kx[t];
}
template <Pipe P>
__device__ __forceinline__ auto vtap(const U8Params& p, int t) {
    if constexpr (P == Pipe::FFMA) return p.kyf[t];   // kyf = ky_q8 * 2^-16: the sums are acc / 65536, still exact
    else return p.ky[t];
}

// ---- DP --------------------------------------------------------------------------------------------------------------------
// When every Q8 tap is a byte (0 .. 255: every kernel with non-negative taps -- Gaussian, box, motion blur) and the horizontal
// sums fit 16 bits (255 * sum(kx) <= 65535), the reference's integer arithmetic maps onto
//   horizontal  dp4a: the 4 pixels of a group are byte-transposed into one word per channel and 4 taps are ONE instruction; a window
//               that starts sh bytes into a word is not shifted into place -- it meets the aligned words with taps delayed by
//               sh bytes (15 taps: 4 or 5 dp4a instead of 15 FMAs);
//   vertical    dp2a: the horizontal sums of two consecutive rows share a register (lo / hi 16 bits) and 2 taps are one
//               instruction (15 taps: 8 dp2a); the pair registers for odd rows are one PRMT from the even ones.
// The ring holds u16 sums (8 B per pixel instead of 16), so two CTAs fit an SM.  Integer sums are order-independent: the results
// are the reference's bits, like the FFMA / IMAD pipelines (which remain for kernels with negative or larger taps).
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
// 16-byte chunk c of a ring row (2 pixels) lives at chunk c ^ ((c >> 3) & 3): the horizontal pass writes 4 consecutive chunks per
// lane (64-byte lane stride), which without the swizzle would hit two bank groups from eight lanes
__device__ __forceinline__ uint32_t dp_chunk(uint32_t c) { return c ^ ((c >> 3) & 3u); }

// H: the horizontal sums of stage row hr, pixels [8 ht, 8 ht + 8), into ring row slot * 8 + hr.
template <int HALF, Pipe P>
__device__ __forceinline__ void h_pass(uint32_t stage, uint32_t ring, int slot, int ht, int hr, const U8Params& p) {
    constexpr int K = 2 * HALF + 1;
    constexpr int NLOAD = CHUNK + 2 * HALF;
    // pixels [8*ht - 8, 8*ht + 16) of the strip = 24 words = 6 aligned 16-byte chunks
    uint32_t w[24];
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        const int4 v = lds128_i(stage_px(stage, hr, PAD - 8 + 8 * ht + 4 * q));
        w[4 * q + 0] = (uint32_t)v.x; w[4 * q + 1] = (uint32_t)v.y; w[4 * q + 2] = (uint32_t)v.z; w[4 * q + 3] = (uint32_t)v.w;
    }
    const uint32_t rrow = ring + (uint32_t)((slot * CHUNK + hr) * ring_row_bytes(P));
    if constexpr (P == Pipe::DP) {
        // byte transpose: T[c][g] = channel c of pixels 4g .. 4g + 3; T[c][6] = 0 pads the 17-tap window
        uint32_t T[4][7];
#pragma unroll
        for (int g = 0; g < 6; ++g) {
            const uint32_t rg01 = __byte_perm(w[4 * g], w[4 * g + 1], 0x5140), rg23 = __byte_perm(w[4 * g + 2], w[4 * g + 3], 0x5140);
            const uint32_t ba01 = __byte_perm(w[4 * g], w[4 * g + 1], 0x7362), ba23 = __byte_perm(w[4 * g + 2], w[4 * g + 3], 0x7362);
            T[0][g] = __byte_perm(rg01, rg23, 0x5410);
            T[1][g] = __byte_perm(rg01, rg23, 0x7632);
            T[2][g] = __byte_perm(ba01, ba23, 0x5410);
            T[3][g] = __byte_perm(ba01, ba23, 0x7632);
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) T[c][6] = 0u;
        uint32_t hsum[4][8];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
#pragma unroll
            for (int o = 0; o < 8; ++o) {
                const int start = 8 - HALF + o;   // byte of T[c] where output o's window begins
                const int sh = start & 3, j0 = start >> 2;
                uint32_t acc = 0;
#pragma unroll
                for (int q = 0; q < (K + sh + 3) / 4; ++q) acc = __dp4a(T[c][j0 + q], p.kxs[sh][q], acc);   // the taps move, not the pixels
                hsum[c][o] = acc;   // <= 255 * sum(kx) <= 65535
            }
        }
        // 2 pixels per 16-byte chunk: (c0 | c1 << 16, c2 | c3 << 16) per pixel
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            int4 v;
            v.x = (int)__byte_perm(hsum[0][2 * q], hsum[1][2 * q], 0x5410);
            v.y = (int)__byte_perm(hsum[2][2 * q], hsum[3][2 * q], 0x5410);
            v.z = (int)__byte_perm(hsum[0][2 * q + 1], hsum[1][2 * q + 1], 0x5410);
            v.w = (int)__byte_perm(hsum[2][2 * q + 1], hsum[3][2 * q + 1], 0x5410);
            sts128_i(rrow + dp_chunk((uint32_t)(4 * ht + q)) * 16u, v);
        }
    } else {
        Acc4<P> acc[8];
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = Acc4<P>{};
#pragma unroll
        for (int j = 0; j < NLOAD; ++j) {
            const Acc4<P> px = unpack_px<P>(w[8 - HALF + j]);
#pragma unroll
            for (int o = 0; o < 8; ++o) {
                const int ti = j - o;
                if (ti >= 0 && ti < K) mac4(acc[o], px, htap<P>(p, ti));
            }
        }
        // lane ht's 8 pixels are 128 contiguous bytes, their 16-byte chunks swizzled by ht & 7
#pragma unroll
        for (int o = 0; o < 8; ++o) sts_acc<P>(rrow + (uint32_t)ht * 128u + ((((uint32_t)o) ^ ((uint32_t)ht & 7u)) << 4), acc[o]);
    }
}

// Output chunk c of unit u, strip column vx: px(o) goes to row ra + 8c + o, for the rows and the column inside the image.
template <typename F>
__device__ __forceinline__ void store_column(const Unit& u, int c, int vx, const U8Params& p, F px) {
    const int x = u.x0 + vx;
    if (x < p.cols) {
        const int yb = u.ra + CHUNK * c;
        uint32_t* out = p.dst + (size_t)yb * p.dst_pitch_px + x;
#pragma unroll
        for (int o = 0; o < 8; ++o)
            if (yb + o < u.rb) __stcs(out + (size_t)o * p.dst_pitch_px, px(o));
    }
}

// V: output chunk c of unit u in strip column vx, from the ring rows that hold the horizontal sums of chunks c .. c + 2.
template <int HALF, Pipe P>
__device__ __forceinline__ void v_pass(uint32_t ring, int c, int vx, const Unit& u, const U8Params& p) {
    constexpr int K = 2 * HALF + 1;
    constexpr int NLOAD = CHUNK + 2 * HALF;   // rows a vertical window block reads
    const uint32_t cbase = (uint32_t)((c % 3) * CHUNK);
    if constexpr (P == Pipe::DP) {
        constexpr int NP = HALF + 1;          // tap pairs
        const uint32_t v_off = dp_chunk((uint32_t)vx >> 1) * 16u + ((uint32_t)vx & 1u) * 8u;
        uint32_t w01[NLOAD], w23[NLOAD];   // (c0 | c1 << 16), (c2 | c3 << 16) of window rows 0 .. NLOAD - 1
#pragma unroll
        for (int j = 0; j < NLOAD; ++j) {
            uint32_t sr = cbase + (uint32_t)(8 - HALF + j);
            if (sr >= RING_ROWS) sr -= RING_ROWS;
            const uint2 v = lds64(ring + sr * (uint32_t)ring_row_bytes(P) + v_off);
            w01[j] = v.x;
            w23[j] = v.y;
        }
        uint32_t px[8];
#pragma unroll
        for (int o = 0; o < 8; ++o) px[o] = 0u;
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            // pair registers: E[m] = (row 2m, row 2m + 1), O[m] = (row 2m + 1, row 2m + 2) of this channel
            const uint32_t sel = (ch & 1) ? 0x7632u : 0x5410u;
            uint32_t E[HALF + 4], O[HALF + 4];
#pragma unroll
            for (int m = 0; m < HALF + 4; ++m) {
                constexpr int last = NLOAD - 1;
                const int r0 = 2 * m, r1 = 2 * m + 1, r2 = (2 * m + 2) > last ? last : (2 * m + 2);   // a row beyond the window only meets a zero tap
                const uint32_t a0 = ch < 2 ? w01[r0] : w23[r0], a1 = ch < 2 ? w01[r1] : w23[r1], a2 = ch < 2 ? w01[r2] : w23[r2];
                E[m] = __byte_perm(a0, a1, sel);
                O[m] = __byte_perm(a1, a2, sel);
            }
#pragma unroll
            for (int o = 0; o < 8; ++o) {
                uint32_t acc = 0;
#pragma unroll
                for (int t = 0; t < NP; ++t) {
                    const uint32_t pr = (o & 1) ? O[(o - 1) / 2 + t] : E[o / 2 + t];   // rows (o + 2t, o + 2t + 1)
                    acc = (t & 1) ? __dp2a_hi(pr, p.ky4[t >> 1], acc) : __dp2a_lo(pr, p.ky4[t >> 1], acc);
                }
                // divClampU8(65536) for acc >= 0: trunc((acc + 32768) / 65536), at most 255.99.. -> clamp
                const uint32_t q = min((acc + 32768u) >> 16, 255u);
                px[o] |= q << (8 * ch);
            }
        }
        store_column(u, c, vx, p, [&](int o) { return px[o]; });
    } else {
        // pixel vx's 16 bytes in a ring row, with the chunk swizzle of h_pass
        const uint32_t v_col = ring + ((uint32_t)vx >> 3) * 128u + ((((uint32_t)vx & 7u) ^ (((uint32_t)vx >> 3) & 7u)) << 4);
        Acc4<P> acc[8];
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = Acc4<P>{};
#pragma unroll
        for (int j = 0; j < NLOAD; ++j) {
            uint32_t sr = cbase + (uint32_t)(8 - HALF + j);
            if (sr >= RING_ROWS) sr -= RING_ROWS;
            const Acc4<P> v = lds_acc<P>(v_col + sr * (uint32_t)ring_row_bytes(P));
#pragma unroll
            for (int o = 0; o < 8; ++o) {
                const int ti = j - o;
                if (ti >= 0 && ti < K) mac4(acc[o], v, vtap<P>(p, ti));
            }
        }
        store_column(u, c, vx, p, [&](int o) { return pack_rgba(acc[o]); });
    }
}

template <int HALF, Pipe P>
__global__ void __launch_bounds__(NTHREADS, ctas_per_sm(P)) fused_sep_rgba8_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ U8Params p) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t ring = smem0 + NSTAGE * STAGE_BYTES;
    const uint32_t bar0 = ring + RING_ROWS * ring_row_bytes(P);
    const int tid = threadIdx.x;
    const int n_units = p.n_strips * p.n_bands;

    int pu = blockIdx.x, pi = 0;
    uint32_t pcount = 0;
    auto produce = [&]() {
        if (pu >= n_units) return;
        const Unit u = decode_unit(pu, p);
        const uint32_t st = pcount % NSTAGE;
        fence_proxy_async();
        mbar_arrive_expect_tx(bar0 + 8 * st, STAGE_BYTES);
        tma_load_2d(smem0 + st * STAGE_BYTES, &tmap, u.x0 - PAD, u.ra - CHUNK + CHUNK * pi, bar0 + 8 * st);
        tma_load_2d(smem0 + st * STAGE_BYTES + BLOCK_BYTES, &tmap, u.x0 - PAD + BW, u.ra - CHUNK + CHUNK * pi, bar0 + 8 * st);
        ++pcount;
        if (++pi == u.n_in) { pi = 0; pu += gridDim.x; }
    };
    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap) : "memory");
        for (int i = 0; i < NSTAGE; ++i) mbar_init(bar0 + 8 * i, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0)
        for (int i = 0; i < NSTAGE; ++i) produce();

    const int ht = tid & 31, hr = tid >> 5;
    uint32_t ccount = 0;
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const Unit u = decode_unit(unit, p);
        const int xs0 = u.x0 - PAD;

        for (int i = 0; i < u.n_in; ++i, ++ccount) {
            const uint32_t st = ccount % NSTAGE;
            const uint32_t stage = smem0 + st * STAGE_BYTES;
            while (!mbar_try_wait(bar0 + 8 * st, (ccount / NSTAGE) & 1u)) {}
            const int y0 = u.ra - CHUNK + CHUNK * i;
            const bool fix_r = p.fix && (y0 < 0 || y0 + CHUNK > p.rows);
            const bool fix_x = p.fix && (xs0 < 0 || xs0 + SW > p.cols);
            if (fix_r || fix_x) {
                fixup_stage_u8(stage, y0, xs0, fix_x, fix_r, p);
                __syncthreads();
            }
            h_pass<HALF, P>(stage, ring, i % 3, ht, hr, p);
            __syncthreads();
            if (tid == 0) produce();
            if (i >= 2) v_pass<HALF, P>(ring, i - 2, tid, u, p);
            __syncthreads();
        }
    }
}

template <int HALF>
int launch_u8(Pipe P, const CUtensorMap& tmap, const U8Params& p, int n_units, int sm_count, cudaStream_t s) {
    auto k = P == Pipe::DP     ? fused_sep_rgba8_kernel<HALF, Pipe::DP>
             : P == Pipe::FFMA ? fused_sep_rgba8_kernel<HALF, Pipe::FFMA>
                               : fused_sep_rgba8_kernel<HALF, Pipe::IMAD>;
    const int smem = smem_bytes(P);
    const int max_grid = ctas_per_sm(P) * sm_count;   // persistent CTAs
    ZB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k<<<n_units < max_grid ? n_units : max_grid, NTHREADS, smem, s>>>(tmap, p);
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace

int conv_separable_fused_rgba8(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border,
                               cudaStream_t s, int row0, int row1) {
    const int half_x = nx / 2, half_y = ny / 2;
    const int half = half_x > half_y ? half_x : half_y;
    if (half < 1 || half > MAX_HALF) return ZB_ERR_UNSUPPORTED;
    if (src->cols < 16 || src->rows < 16) return ZB_ERR_UNSUPPORTED;
    if (images_overlap(src, dst, 4)) return ZB_ERR_UNSUPPORTED;   // in place / overlapping views: the temp-plane path
    if (((uintptr_t)src->data & 15u) || (src->stride & 3u)) return ZB_ERR_UNSUPPORTED;  // TMA: 16-byte aligned base and row pitch
    U8Params p;
    memset(&p, 0, sizeof(p));
    long long sax = 0, say = 0;
    for (int i = 0; i < nx; ++i) { const int q = (int)roundf(kx[i] * 256.0f); p.kx[i + (half - half_x)] = q; sax += llabs((long long)q); }
    for (int i = 0; i < ny; ++i) { const int q = (int)roundf(ky[i] * 256.0f); p.ky[i + (half - half_y)] = q; say += llabs((long long)q); }
    if (sax * 255 * say + 32768 >= 2147483647LL) return ZB_ERR_UNSUPPORTED;  // i32 accumulators must be provably safe
    const bool fmath = (sax * 255 * say <= (1LL << 24)) && g_tune_u8_fmath.load() != 0;  // f32 is exact up to 2^24
    for (int i = 0; i < MAXK; ++i) { p.kxf[i] = (float)p.kx[i]; p.kyf[i] = (float)p.ky[i] * (1.0f / 65536.0f); }   // exact power-of-two scaling
    EncodeTiledFn encode = encode_tiled_fn();
    if (!encode) return ZB_ERR_UNSUPPORTED;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (di.smem_optin < (size_t)smem_bytes(Pipe::IMAD)) return ZB_ERR_UNSUPPORTED;
    p.src = (const uint32_t*)src->data;
    p.dst = (uint32_t*)dst->data;
    p.src_pitch_px = src->stride;
    p.dst_pitch_px = dst->stride;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.border = border;
    p.n_strips = (p.cols + TW - 1) / TW;
    p.row0 = row0 < 0 ? 0 : row0;
    p.row1 = (row1 < 0 || row1 > p.rows) ? p.rows : row1;
    if (p.row1 <= p.row0) return ZB_OK;
    const BandPlan plan = plan_bands(p.row1 - p.row0, p.n_strips, di.sm_count);
    p.band_rows = plan.band_rows;
    p.n_bands = plan.n_bands;
    p.fix = border != ZB_BORDER_ZERO;

    CUtensorMap tmap;
    const cuuint64_t gdim[2] = {(cuuint64_t)p.cols, (cuuint64_t)p.rows};
    const cuuint64_t gstr[1] = {(cuuint64_t)src->stride * 4};
    const cuuint32_t box[2] = {(cuuint32_t)BW, (cuuint32_t)CHUNK};
    const cuuint32_t estr[2] = {1, 1};
    CUresult cr = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, src->data, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
        snprintf(t_last_error, sizeof(t_last_error), "cuTensorMapEncodeTiled (rgba8) failed: %d", (int)cr);
        return ZB_ERR_UNSUPPORTED;
    }
    // DP pipeline: every tap a byte (non-negative), horizontal sums within 16 bits
    bool dp = g_tune_u8_dp.load() != 0 && sax * 255 <= 65535;
    for (int i = 0; i < MAXK && dp; ++i) dp = p.kx[i] >= 0 && p.kx[i] <= 255 && p.ky[i] >= 0 && p.ky[i] <= 255;
    if (dp) {
        // taps k[4q + b - sh] in byte b of word q, zero outside the kernel
        auto tap_word = [](const int* k, int q, int sh) {
            unsigned word = 0;
            for (int b = 0; b < 4; ++b) {
                const int t = 4 * q + b - sh;
                if (t >= 0 && t < MAXK) word |= (unsigned)k[t] << (8 * b);
            }
            return word;
        };
        for (int q = 0; q < 5; ++q) {
            p.ky4[q] = tap_word(p.ky, q, 0);
            for (int sh = 0; sh < 4; ++sh) p.kxs[sh][q] = tap_word(p.kx, q, sh);
        }
    }
    const Pipe pipe = dp ? Pipe::DP : fmath ? Pipe::FFMA : Pipe::IMAD;
    t_last_kernel = dp ? "fused_sep_rgba8_dp" : fmath ? "fused_sep_rgba8_f" : "fused_sep_rgba8";
    const int n_units = p.n_strips * p.n_bands;
    switch (half) {
        case 1: return launch_u8<1>(pipe, tmap, p, n_units, di.sm_count, s);
        case 2: return launch_u8<2>(pipe, tmap, p, n_units, di.sm_count, s);
        case 3: return launch_u8<3>(pipe, tmap, p, n_units, di.sm_count, s);
        case 4: return launch_u8<4>(pipe, tmap, p, n_units, di.sm_count, s);
        case 5: return launch_u8<5>(pipe, tmap, p, n_units, di.sm_count, s);
        case 6: return launch_u8<6>(pipe, tmap, p, n_units, di.sm_count, s);
        case 7: return launch_u8<7>(pipe, tmap, p, n_units, di.sm_count, s);
        case 8: return launch_u8<8>(pipe, tmap, p, n_units, di.sm_count, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

}  // namespace zb
