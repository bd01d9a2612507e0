// zb_conv_tile_u8.cu -- single-pass separable convolution for 8-bit images of ANY channel count (gray, Rgb, Rgba) and any
// alignment, border mode and view stride: the fallback between the TMA kernel (zb_conv_fused_u8.cu: Rgba only, 16-byte
// friendly) and the two-pass path (zb_conv_generic.cu: i32 temp plane through HBM, 10 bytes of traffic per byte of image).
//
// Reference semantics (convolution.zig:340-431, :441-647): Q8 taps round(k*256), horizontal pass into an i32 temp (not
// rounded), vertical pass, one divClampU8(65536).  Integer sums are order-independent, so the tile decomposition changes no bit
// as long as nothing overflows; the host proves that for i32 (otherwise the two-pass path with i64 accumulators runs).
//
// A row of interleaved pixels is treated as a stream of BYTES: output byte b of a row is sum_i in[b + CH*(i - half)] * kx[i],
// i.e. the channel structure is nothing but a tap stride of CH bytes.  One CTA produces a TH-row x 256-byte tile:
//   load : (TH + 2*half) rows x (256 + 2*half*CH) bytes into shared memory, border-resolved per pixel (resolveIndex);
//   H    : a thread produces runs of 8 consecutive bytes of a tile row from one set of 64-bit loads; every tap is a compile-time
//          byte extract + integer multiply-add with the tap as an immediate constant-bank operand (the kernel is specialised on
//          `half`); results go to an i32 tile in shared memory;
//   V    : thread t owns byte column t and walks down it with a K-deep register window (one shared load per output row),
//          divClampU8, byte store.
// HBM traffic: ~1.3 bytes read + 1 written per image byte.
#include <cstdlib>

#include "zb_conv.h"
#include "zb_device.cuh"

namespace zb {

namespace {

constexpr int TWB = 256;          // output bytes per tile row = threads per CTA
constexpr int TU_MAX_HALF = 15;
constexpr int DP_TH = 48;               // rows per tile of the dot-product variant: 48 KB of shared memory -> four CTAs per SM
constexpr int TU_DP_MAX_HALF = 8;        // the dot-product variant: registers of the vertical window, 16 tap words per output byte

struct TileParams {
    int kx[2 * TU_MAX_HALF + 1];   // taps aligned to the common half-width (zero padded)
    int ky[2 * TU_MAX_HALF + 1];
    const uint8_t* src;
    uint8_t* dst;
    size_t src_pitch, dst_pitch;   // bytes
    int rows, cols, row_bytes, border;
    // DP variant: horizontal tap words tw[m][j] = the four Q8 taps (bytes) that output byte m of an 8-byte run applies to bytes
    // 4j .. 4j + 3 of the run's span; vertical tap pairs for even (kye) and odd (kyo) output rows
    uint32_t tw[8][20];
    uint32_t kye[TU_DP_MAX_HALF + 1], kyo[TU_DP_MAX_HALF + 1];
    int dst_word_ok;               // dst base and pitch are multiples of 4: the vertical pass stores whole words
    int src_word_ok;               // src base, pitch and row length are multiples of 4: interior tiles load whole words
    int no_clamp;                  // 255 * sum(kx) * sum(ky) + 32768 < 2^24: divClampU8 never clamps
    int k2[49];                    // dense variant: Q8 taps of the (2 HALF + 1)^2 square the kernel is centred in (zero padded)
    int dst_dword_ok;              // dst base and pitch are multiples of 8: the dense kernel stores 8 bytes at once
};

// Load stage shared by both tile kernels: in[tr][tb] = source byte at row resolve(y0 + tr - HALF), byte position
// (b0 + tb - HALF*CH), border-resolved per pixel.
template <int CH, int HALF, int IR, int IW>
__device__ __forceinline__ void tile_load(const TileParams& p, uint8_t* in, int t, int b0, int y0) {
    // Interior tiles of a 4-byte aligned image (base, pitch and row length): no pixel needs the border rule, so the tile is copied
    // as 32-bit words -- two aligned loads (the second one a neighbour's first: an L1 hit) and a funnel shift per word, since a
    // tile row starts HALF * CH bytes before a 256-byte boundary.
    {
        const int g0 = b0 - HALF * CH;                 // first byte of the tile row within the source row
        if (p.src_word_ok && g0 >= 0 && g0 + IW <= p.row_bytes && y0 - HALF >= 0 && y0 - HALF + IR <= p.rows) {
            constexpr int WPR = IW / 4;                // words per tile row
            constexpr int UB = 4;                      // rows in flight per thread
            // thread -> (word column tx [+ 64], rows ty, ty + 4, ...): no division, one pointer step per row
            const int tx = t & 63, ty = t >> 6;
            const uint8_t* base = p.src + (size_t)(y0 - HALF) * p.src_pitch + g0;
#pragma unroll
            for (int cq = 0; cq < (WPR + 63) / 64; ++cq) {
                const int wq = tx + 64 * cq;
                if (wq < WPR) {
                    const uintptr_t a0 = (uintptr_t)(base + 4 * wq) + (size_t)ty * p.src_pitch;
                    const unsigned sh = (unsigned)(a0 & 3u) * 8u;      // pitch is a multiple of 4: the same shift for every row
                    const uint32_t* q = reinterpret_cast<const uint32_t*>(a0 & ~(uintptr_t)3);
                    const size_t step = p.src_pitch;                    // bytes per row; 4 rows per iteration of this thread
                    uint32_t* d = reinterpret_cast<uint32_t*>(in + ty * IW + 4 * wq);
                    for (int tr0 = ty; tr0 < IR; tr0 += 4 * UB) {
                        uint32_t lo[UB], hi[UB];
#pragma unroll
                        for (int u = 0; u < UB; ++u) {
                            lo[u] = hi[u] = 0u;
                            if (tr0 + 4 * u < IR) {
                                const uint32_t* qq = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(q) + (size_t)(4 * u) * step);
                                lo[u] = __ldg(qq);
                                if (sh) hi[u] = __ldg(qq + 1);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < UB; ++u)
                            if (tr0 + 4 * u < IR) d[(4 * u) * (IW / 4)] = __funnelshift_r(lo[u], hi[u], sh);
                        q = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(q) + (size_t)(4 * UB) * step);
                        d += (4 * UB) * (IW / 4);
                    }
                }
            }
            return;
        }
    }
    // LB rows are fetched per batch so that 2*LB independent global loads are in flight before the first shared-memory store
    // (one load per iteration would expose the full memory latency IR times per tile).
    {
        constexpr int LB = 8;
        constexpr int NCOL = (IW + TWB - 1) / TWB;   // byte columns per thread (2)
        // the pixel / channel of this thread's byte columns and where the border sends them: row independent, computed once
        int gcol[NCOL];    // resolved byte position inside a source row, or -1 (zero)
#pragma unroll
        for (int k = 0; k < NCOL; ++k) {
            const int tb = t + k * TWB;
            const int gb = b0 + tb - HALF * CH;
            int g = -1;
            if (tb < IW) {
                if (gb >= 0 && gb < p.row_bytes) {
                    g = gb;
                } else {
                    const int px = gb >= 0 ? gb / CH : -((-gb + CH - 1) / CH);     // floor division
                    const int chn = gb - px * CH;
                    const int rx = resolve_index(px, p.cols, p.border);
                    if (rx >= 0) g = rx * CH + chn;
                }
            }
            gcol[k] = g;
        }
        for (int tr0 = 0; tr0 < IR; tr0 += LB) {
            uint8_t v[LB][NCOL];
#pragma unroll
            for (int u = 0; u < LB; ++u) {
                const int tr = tr0 + u;
                const int ry = tr < IR ? resolve_index(y0 + tr - HALF, p.rows, p.border) : -1;
                const uint8_t* rowp = p.src + (size_t)(ry < 0 ? 0 : ry) * p.src_pitch;
#pragma unroll
                for (int k = 0; k < NCOL; ++k) v[u][k] = (ry >= 0 && gcol[k] >= 0) ? __ldg(rowp + gcol[k]) : (uint8_t)0;
            }
#pragma unroll
            for (int u = 0; u < LB; ++u) {
                const int tr = tr0 + u;
                if (tr < IR) {
#pragma unroll
                    for (int k = 0; k < NCOL; ++k)
                        if (t + k * TWB < IW) in[tr * IW + t + k * TWB] = v[u][k];
                }
            }
        }
    }
}

template <int CH, int HALF>
__global__ void __launch_bounds__(TWB) sep_tile_u8_kernel(const __grid_constant__ TileParams p) {
    constexpr int K = 2 * HALF + 1;
    constexpr int TH = HALF <= 7 ? 64 : 32;                 // output rows per tile
    constexpr int IR = TH + 2 * HALF;                       // tile rows held in shared memory
    constexpr int IW = (TWB + 2 * HALF * CH + 7) & ~7;      // input bytes per tile row (8-byte granular: 64-bit loads in the H pass)
    extern __shared__ __align__(16) unsigned char smem[];
    int* tmp = reinterpret_cast<int*>(smem);                // [IR][TWB] horizontal sums
    uint8_t* in = smem + (size_t)IR * TWB * sizeof(int);    // [IR][IW]  border-resolved source bytes
    const int t = threadIdx.x;
    const int b0 = blockIdx.x * TWB;                        // first output byte of the tile within a row
    const int y0 = ZB_GRID_ROW() * TH;                      // first output row
    if (y0 >= p.rows) return;   // past the last tile (uniform per block)

    tile_load<CH, HALF, IR, IW>(p, in, t, b0, y0);
    __syncthreads();

    // ---- horizontal pass: tmp[tr][b] = sum_i in[tr][b + i*CH] * kx[i].  A thread produces a run of 8 consecutive bytes of one tile
    // row from ONE set of 64-bit shared-memory loads (the 8 + 2*HALF*CH bytes the run touches); every tap byte is then a compile-time
    // byte extract.  9x fewer shared-memory instructions than one byte load per tap, which is what bounded the first version.
    {
        constexpr int SPAN = 8 + 2 * HALF * CH;          // bytes a run reads
        constexpr int NQ = (SPAN + 7) / 8;               // 64-bit words
        for (int idx = t; idx < IR * (TWB / 8); idx += TWB) {
            const int tr = idx / (TWB / 8), run = idx % (TWB / 8);
            const unsigned long long* q = reinterpret_cast<const unsigned long long*>(in + tr * IW + 8 * run);
            unsigned long long w[NQ];
#pragma unroll
            for (int i = 0; i < NQ; ++i) w[i] = (8 * run + 8 * i < IW) ? q[i] : 0ull;
            int acc[8];
#pragma unroll
            for (int m = 0; m < 8; ++m) acc[m] = 0;
#pragma unroll
            for (int i = 0; i < K; ++i)
#pragma unroll
                for (int m = 0; m < 8; ++m) {
                    const int o = m + i * CH;   // byte offset inside the span: static
                    acc[m] += (int)((w[o >> 3] >> (8 * (o & 7))) & 0xFFull) * p.kx[i];
                }
            int4* dsts = reinterpret_cast<int4*>(tmp + tr * TWB + 8 * run);
            dsts[0] = make_int4(acc[0], acc[1], acc[2], acc[3]);
            dsts[1] = make_int4(acc[4], acc[5], acc[6], acc[7]);
        }
    }
    __syncthreads();

    // ---- vertical pass: out[y0 + r][b0 + t] = divClampU8(sum_j tmp[r + j][t] * ky[j], 65536); thread t walks down byte column t
    if (b0 + t < p.row_bytes) {
        const int nrows = min(TH, p.rows - y0);
        uint8_t* out = p.dst + (size_t)y0 * p.dst_pitch + (size_t)(b0 + t);
        if constexpr (K <= 15) {
            // sliding window in registers: one new shared-memory value per output row instead of K (unrolled K-fold so that the
            // rotating window indices are compile-time)
            int win[K];
#pragma unroll
            for (int j = 0; j < K - 1; ++j) win[j] = tmp[j * TWB + t];
            for (int r0 = 0; r0 < nrows; r0 += K) {
#pragma unroll
                for (int rr = 0; rr < K; ++rr) {
                    const int r = r0 + rr;
                    if (r < nrows) {
                        win[(rr + K - 1) % K] = tmp[(r + K - 1) * TWB + t];
                        int acc = 0;
#pragma unroll
                        for (int j = 0; j < K; ++j) acc += win[(rr + j) % K] * p.ky[j];
                        out[(size_t)r * p.dst_pitch] = div_clamp_u8<int>(acc, 65536);
                    }
                }
            }
        } else {
#pragma unroll 2
            for (int r = 0; r < nrows; ++r) {
                const int* q = tmp + r * TWB + t;
                int acc = 0;
#pragma unroll
                for (int j = 0; j < K; ++j) acc += q[j * TWB] * p.ky[j];
                out[(size_t)r * p.dst_pitch] = div_clamp_u8<int>(acc, 65536);
            }
        }
    }
}

template <int CH, int HALF>
int launch_tile(const TileParams& p, cudaStream_t s) {
    constexpr int TH = HALF <= 7 ? 64 : 32;
    constexpr int IR = TH + 2 * HALF;
    constexpr int IW = (TWB + 2 * HALF * CH + 7) & ~7;
    constexpr int smem = IR * TWB * (int)sizeof(int) + IR * IW;
    auto k = sep_tile_u8_kernel<CH, HALF>;
    if (smem > 48 * 1024) ZB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const dim3 grid = row_grid(div_up((size_t)p.row_bytes, TWB), div_up((size_t)p.rows, TH));
    k<<<grid, TWB, smem, s>>>(p);
    ZB_LAUNCHED();
    return ZB_OK;
}

// ================================================================================================
// DP variant (every Q8 tap a byte 0 .. 255 and 255 * sum(kx) <= 65535: Gaussian, box, motion blur): the same tile on the
// integer dot-product instructions.
//   H : a thread produces 8 consecutive bytes of TWO tile rows.  Output byte m is sum_j dp4a(W_j, tw[m][j]) over the aligned
//       32-bit words W_j of the run's span: instead of shifting the pixels into place for every output, the host shifts the TAPS
//       (tw[m][j] holds the taps that fall on bytes 4j .. 4j + 3 for output m; words without a tap are skipped at compile time).
//       Gray: 4-5 dp4a per output byte instead of 15 extract + multiply-add triples; Rgb: 11-12.  The sums (<= 65535) of the two
//       rows share a word: tmp[pair][byte] = row 2 pair | row 2 pair + 1 << 16.
//   V : a thread owns 4 byte columns x TH/4 rows with the pairs it needs in registers; an even output row is HALF + 1 dp2a over
//       the pairs with taps (ky0, ky1), (ky2, ky3), ..., an odd one the same pairs with taps (0, ky0), (ky1, ky2), ... -- again the
//       taps move, not the data.  divClampU8(65536) of a non-negative sum = min((acc + 32768) >> 16, 255); word stores.
// Integer sums are order-independent: same bits as the reference (and as the IMAD variant above, which stays for other kernels).
// ================================================================================================
template <int CH, int HALF>
__global__ void __launch_bounds__(TWB, 4) sep_tile_u8_dp_kernel(const __grid_constant__ TileParams p) {
    constexpr int K = 2 * HALF + 1;
    constexpr int TH = DP_TH;
    constexpr int IR = TH + 2 * HALF;                       // even
    constexpr int IW = (TWB + 2 * HALF * CH + 7) & ~7;
    constexpr int NPAIR = IR / 2;
    extern __shared__ __align__(16) unsigned char smem[];
    uint32_t* tmp = reinterpret_cast<uint32_t*>(smem);                  // [NPAIR][TWB] horizontal sums of rows (2 pr, 2 pr + 1)
    uint8_t* in = smem + (size_t)NPAIR * TWB * sizeof(uint32_t);        // [IR][IW]
    const int t = threadIdx.x;
    const int b0 = blockIdx.x * TWB;
    const int y0 = ZB_GRID_ROW() * TH;
    if (y0 >= p.rows) return;   // past the last tile (uniform per block)
    tile_load<CH, HALF, IR, IW>(p, in, t, b0, y0);
    __syncthreads();

    {
        constexpr int SPAN = 8 + 2 * HALF * CH;          // bytes a run reads
        constexpr int NQ = (SPAN + 7) / 8;               // 64-bit words
        constexpr int NW = (SPAN + 3) / 4;               // 32-bit words
        static_assert(NW <= 20, "tap word table");
        for (int idx = t; idx < NPAIR * (TWB / 8); idx += TWB) {
            const int pr = idx / (TWB / 8), run = idx % (TWB / 8);
            uint32_t acc[2][8];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const unsigned long long* q = reinterpret_cast<const unsigned long long*>(in + (2 * pr + h) * IW + 8 * run);
                unsigned long long w[NQ];
#pragma unroll
                for (int i = 0; i < NQ; ++i) w[i] = (8 * run + 8 * i < IW) ? q[i] : 0ull;
#pragma unroll
                for (int m = 0; m < 8; ++m) {
                    uint32_t a = 0;
#pragma unroll
                    for (int j = 0; j < NW; ++j) {
                        // does a tap of output m fall on bytes 4j .. 4j + 3 of the span?  (compile time after unrolling)
                        bool has = false;
#pragma unroll
                        for (int b = 4 * j; b < 4 * j + 4; ++b) has = has || (b >= m && (b - m) % CH == 0 && (b - m) / CH < K);
                        if (has) a = __dp4a((uint32_t)(w[j >> 1] >> (32 * (j & 1))), p.tw[m][j], a);
                    }
                    acc[h][m] = a;
                }
            }
            uint4* dsts = reinterpret_cast<uint4*>(tmp + pr * TWB + 8 * run);
            dsts[0] = make_uint4(acc[0][0] | (acc[1][0] << 16), acc[0][1] | (acc[1][1] << 16), acc[0][2] | (acc[1][2] << 16), acc[0][3] | (acc[1][3] << 16));
            dsts[1] = make_uint4(acc[0][4] | (acc[1][4] << 16), acc[0][5] | (acc[1][5] << 16), acc[0][6] | (acc[1][6] << 16), acc[0][7] | (acc[1][7] << 16));
        }
    }
    __syncthreads();

    {
        constexpr int RPT = TH / 4;                       // rows per thread (12), produced in strips of RPG rows: a strip's window of
        constexpr int RPG = RPT / 2;                      // row pairs stays in registers (6 rows: 10 pair words x 4 columns)
        constexpr int NE = RPG / 2 + HALF;                // pairs the rows of a strip read
        static_assert(RPG % 2 == 0, "strips start on an even row");
        const int cg = t & 63, rg = t >> 6;
        const int bcol = b0 + 4 * cg;
#pragma unroll 1
        for (int strip = 0; strip < 2; ++strip) {
        const int r0 = rg * RPT + strip * RPG;
        if (bcol < p.row_bytes && y0 + r0 < p.rows) {
            uint4 E[NE];
#pragma unroll
            for (int e = 0; e < NE; ++e) E[e] = *reinterpret_cast<const uint4*>(tmp + (r0 / 2 + e) * TWB + 4 * cg);
            const int nrows = min(RPG, p.rows - y0 - r0);
            uint8_t* out = p.dst + (size_t)(y0 + r0) * p.dst_pitch + (size_t)bcol;
            const int nb = min(4, p.row_bytes - bcol);
            // one output word: 4 byte columns of row rr; the sums start at 32768 (the rounding of divClampU8)
            auto row_sums = [&](int rr, uint32_t& a0, uint32_t& a1, uint32_t& a2, uint32_t& a3) {
                a0 = a1 = a2 = a3 = 32768u;
#pragma unroll
                for (int q = 0; q <= HALF; ++q) {
                    const uint4 e = E[rr / 2 + q];
                    const uint32_t kt = (rr & 1) ? p.kyo[q] : p.kye[q];
                    a0 = __dp2a_lo(e.x, kt, a0);
                    a1 = __dp2a_lo(e.y, kt, a1);
                    a2 = __dp2a_lo(e.z, kt, a2);
                    a3 = __dp2a_lo(e.w, kt, a3);
                }
            };
            if (nrows == RPG && nb == 4 && p.dst_word_ok && p.no_clamp) {
                // whole strip, word stores, and 255 * sum(kx) * sum(ky) + 32768 < 2^24: the quotient is byte 2 of the sum as it stands
#pragma unroll
                for (int rr = 0; rr < RPG; ++rr) {
                    uint32_t a0, a1, a2, a3;
                    row_sums(rr, a0, a1, a2, a3);
                    *reinterpret_cast<uint32_t*>(out + (size_t)rr * p.dst_pitch) =
                        __byte_perm(__byte_perm(a0, a1, 0x0062), __byte_perm(a2, a3, 0x0062), 0x5410);
                }
            } else {
#pragma unroll
                for (int rr = 0; rr < RPG; ++rr) {
                    if (rr < nrows) {
                        uint32_t a0, a1, a2, a3;
                        row_sums(rr, a0, a1, a2, a3);
                        const uint32_t q0 = min(a0 >> 16, 255u), q1 = min(a1 >> 16, 255u), q2 = min(a2 >> 16, 255u), q3 = min(a3 >> 16, 255u);
                        uint8_t* o = out + (size_t)rr * p.dst_pitch;
                        if (p.dst_word_ok && nb == 4) {
                            *reinterpret_cast<uint32_t*>(o) = q0 | (q1 << 8) | (q2 << 16) | (q3 << 24);
                        } else {
                            o[0] = (uint8_t)q0;
                            if (nb > 1) o[1] = (uint8_t)q1;
                            if (nb > 2) o[2] = (uint8_t)q2;
                            if (nb > 3) o[3] = (uint8_t)q3;
                        }
                    }
                }
            }
        }
        }
    }
}

template <int CH, int HALF>
int launch_tile_dp(const TileParams& p, cudaStream_t s) {
    constexpr int TH = DP_TH;
    constexpr int IR = TH + 2 * HALF;
    constexpr int IW = (TWB + 2 * HALF * CH + 7) & ~7;
    constexpr int smem = (IR / 2) * TWB * (int)sizeof(uint32_t) + IR * IW;
    auto k = sep_tile_u8_dp_kernel<CH, HALF>;
    if (smem > 48 * 1024) ZB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const dim3 grid = row_grid(div_up((size_t)p.row_bytes, TWB), div_up((size_t)p.rows, TH));
    k<<<grid, TWB, smem, s>>>(p);
    ZB_LAUNCHED();
    return ZB_OK;
}

template <int CH>
int launch_half_dp(int half, const TileParams& p, cudaStream_t s) {
    switch (half) {
        case 1: return launch_tile_dp<CH, 1>(p, s);
        case 2: return launch_tile_dp<CH, 2>(p, s);
        case 3: return launch_tile_dp<CH, 3>(p, s);
        case 4: return launch_tile_dp<CH, 4>(p, s);
        case 5: return launch_tile_dp<CH, 5>(p, s);
        case 6: return launch_tile_dp<CH, 6>(p, s);
        case 7: return launch_tile_dp<CH, 7>(p, s);
        case 8: return launch_tile_dp<CH, 8>(p, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

template <int CH>
int launch_half(int half, const TileParams& p, cudaStream_t s) {
    switch (half) {
        case 1: return launch_tile<CH, 1>(p, s);
        case 2: return launch_tile<CH, 2>(p, s);
        case 3: return launch_tile<CH, 3>(p, s);
        case 4: return launch_tile<CH, 4>(p, s);
        case 5: return launch_tile<CH, 5>(p, s);
        case 6: return launch_tile<CH, 6>(p, s);
        case 7: return launch_tile<CH, 7>(p, s);
        case 8: return launch_tile<CH, 8>(p, s);
        case 9: return launch_tile<CH, 9>(p, s);
        case 10: return launch_tile<CH, 10>(p, s);
        case 11: return launch_tile<CH, 11>(p, s);
        case 12: return launch_tile<CH, 12>(p, s);
        case 13: return launch_tile<CH, 13>(p, s);
        case 14: return launch_tile<CH, 14>(p, s);
        case 15: return launch_tile<CH, 15>(p, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

// ================================================================================================
// Dense (non-separable) convolution, kernels up to 7 x 7 (Image.convolve, convolution.zig:64-253: Q8 taps, one divClampU8(256)).
// Same byte-stream view and the same tile loader.  A thread produces 8 consecutive bytes of one row: per kernel row it loads the
// run's span as words, extracts every byte ONCE (a PRMT) and reuses it for all the taps that meet it, so a 3 x 3 kernel on Rgba
// costs 16 extracts + 24 multiply-adds per kernel row and 8 output bytes -- the generic kernel resolves the border and unpacks a
// pixel per tap (0.98 ms at 8192^2 Rgba against 0.2x here).  i32 accumulators (the host proves the bound), bit-exact.
// ================================================================================================
template <int CH, int HALF>
__global__ void __launch_bounds__(TWB) dense_tile_u8_kernel(const __grid_constant__ TileParams p) {
    constexpr int K = 2 * HALF + 1;
    constexpr int TH = 32;
    constexpr int IR = TH + 2 * HALF;
    constexpr int IW = (TWB + 2 * HALF * CH + 7) & ~7;
    constexpr int SPAN = 8 + 2 * HALF * CH;
    constexpr int NW = (SPAN + 3) / 4;
    extern __shared__ __align__(16) unsigned char smem[];
    uint8_t* in = smem;                                      // [IR][IW]
    const int t = threadIdx.x;
    const int b0 = blockIdx.x * TWB;
    const int y0 = ZB_GRID_ROW() * TH;
    if (y0 >= p.rows) return;   // past the last tile (uniform per block)
    tile_load<CH, HALF, IR, IW>(p, in, t, b0, y0);
    __syncthreads();
    for (int idx = t; idx < TH * (TWB / 8); idx += TWB) {
        const int r = idx / (TWB / 8), run = idx % (TWB / 8);
        const int bcol = b0 + 8 * run;
        if (y0 + r >= p.rows || bcol >= p.row_bytes) continue;
        int acc[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) acc[m] = 0;
#pragma unroll
        for (int dy = 0; dy < K; ++dy) {
            const uint2* q = reinterpret_cast<const uint2*>(in + (r + dy) * IW + 8 * run);
            uint32_t w[NW + 1];
#pragma unroll
            for (int i = 0; i < (NW + 1) / 2; ++i) {
                const uint2 v = q[i];
                w[2 * i] = v.x;
                w[2 * i + 1] = v.y;
            }
            int bytes[SPAN];
#pragma unroll
            for (int sb = 0; sb < SPAN; ++sb) bytes[sb] = (int)__byte_perm(w[sb >> 2], 0u, 0x4440u | (uint32_t)(sb & 3));
#pragma unroll
            for (int dx = 0; dx < K; ++dx) {
                const int kq = p.k2[dy * K + dx];
#pragma unroll
                for (int m = 0; m < 8; ++m) acc[m] += bytes[m + dx * CH] * kq;
            }
        }
        // divClampU8(acc, 256): round half away from zero, clamp; a negative sum clamps to 0
        uint32_t qv[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) qv[m] = (uint32_t)min(max(acc[m] + 128, 0) >> 8, 255);
        uint8_t* o = p.dst + (size_t)(y0 + r) * p.dst_pitch + (size_t)bcol;
        const int nb = min(8, p.row_bytes - bcol);
        if (p.dst_dword_ok && nb == 8) {
            *reinterpret_cast<uint2*>(o) = make_uint2(qv[0] | (qv[1] << 8) | (qv[2] << 16) | (qv[3] << 24), qv[4] | (qv[5] << 8) | (qv[6] << 16) | (qv[7] << 24));
        } else {
#pragma unroll
            for (int m = 0; m < 8; ++m)
                if (m < nb) o[m] = (uint8_t)qv[m];
        }
    }
}

template <int CH, int HALF>
int launch_dense(const TileParams& p, cudaStream_t s) {
    constexpr int TH = 32;
    constexpr int IR = TH + 2 * HALF;
    constexpr int IW = (TWB + 2 * HALF * CH + 7) & ~7;
    constexpr int smem = IR * IW;
    const dim3 grid = row_grid(div_up((size_t)p.row_bytes, TWB), div_up((size_t)p.rows, TH));
    dense_tile_u8_kernel<CH, HALF><<<grid, TWB, smem, s>>>(p);
    ZB_LAUNCHED();
    return ZB_OK;
}

template <int CH>
int launch_dense_half(int half, const TileParams& p, cudaStream_t s) {
    switch (half) {
        case 1: return launch_dense<CH, 1>(p, s);
        case 2: return launch_dense<CH, 2>(p, s);
        case 3: return launch_dense<CH, 3>(p, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

// ================================================================================================
// Image.sobel on a gray Image(u8) (edges.zig:33-73): two 3 x 3 convolutions with .replicate, magnitude sqrt(gx^2 + gy^2) / 4,
// trunc(clamp(0, 255)).  The reference convolves in f32, but every product and partial sum is a small integer (|g| <= 1020), so
// integer arithmetic gives the same numbers; gx^2 + gy^2 < 2^24 converts to f32 exactly and the square root, the division by 4
// and the truncation are the reference's own f32 operations.  Byte tile as above, a thread per 8 consecutive bytes, every source
// byte extracted once.
// ================================================================================================
// CH = 3 / 4 (Rgb / Rgba input): the loader converts to luma on the way in -- convertColor(u8, px), color.zig:1031-1041:
// (13933 r + 46871 g + 4732 b + 32768) >> 16 -- with the .replicate rule applied to the pixel; the gradient code is the gray one.
template <int CH>
__global__ void __launch_bounds__(TWB) sobel_tile_u8_kernel(const __grid_constant__ TileParams p) {
    constexpr int TH = 32;
    constexpr int IR = TH + 2;
    constexpr int IW = (TWB + 2 + 7) & ~7;
    extern __shared__ __align__(16) unsigned char smem[];
    uint8_t* in = smem;
    const int t = threadIdx.x;
    const int b0 = blockIdx.x * TWB;                 // first output column of the tile (gray bytes == pixels)
    const int y0 = ZB_GRID_ROW() * TH;
    if (y0 >= p.rows) return;   // past the last tile (uniform per block)
    if constexpr (CH == 1) {
        tile_load<1, 1, IR, IW>(p, in, t, b0, y0);
    } else {
        for (int idx = t; idx < IR * IW; idx += TWB) {
            const int tr = idx / IW, tb = idx - tr * IW;
            const int y = min(max(y0 + tr - 1, 0), p.rows - 1), x = min(max(b0 + tb - 1, 0), p.cols - 1);   // .replicate
            const uint8_t* q = p.src + (size_t)y * p.src_pitch + (size_t)x * CH;
            const int v = (13933 * (int)q[0] + 46871 * (int)q[1] + 4732 * (int)q[2] + 32768) >> 16;
            in[idx] = (uint8_t)min(max(v, 0), 255);
        }
    }
    __syncthreads();
    for (int idx = t; idx < TH * (TWB / 8); idx += TWB) {
        const int r = idx / (TWB / 8), run = idx % (TWB / 8);
        const int bcol = b0 + 8 * run;
        if (y0 + r >= p.rows || bcol >= p.row_bytes) continue;
        int px[3][10];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const uint2* q = reinterpret_cast<const uint2*>(in + (r + dy) * IW + 8 * run);
            const uint2 a = q[0], b = q[1];
            const uint32_t w[3] = {a.x, a.y, b.x};
#pragma unroll
            for (int sb = 0; sb < 10; ++sb) px[dy][sb] = (int)__byte_perm(w[sb >> 2], 0u, 0x4440u | (uint32_t)(sb & 3));
        }
        uint32_t qv[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const int gx = (px[0][m + 2] - px[0][m]) + 2 * (px[1][m + 2] - px[1][m]) + (px[2][m + 2] - px[2][m]);            // edges.zig:14-18
            const int gy = (px[2][m] + 2 * px[2][m + 1] + px[2][m + 2]) - (px[0][m] + 2 * px[0][m + 1] + px[0][m + 2]);      // :21-25
            const float mag = __fsqrt_rn((float)(gx * gx + gy * gy));
            qv[m] = (uint32_t)(int)fminf(__fmul_rn(mag, 0.25f), 255.0f);   // >= 0 by construction; x / 4 == x * 0.25 exactly
        }
        uint8_t* o = p.dst + (size_t)(y0 + r) * p.dst_pitch + (size_t)bcol;
        const int nb = min(8, p.row_bytes - bcol);
        if (p.dst_dword_ok && nb == 8) {
            *reinterpret_cast<uint2*>(o) = make_uint2(qv[0] | (qv[1] << 8) | (qv[2] << 16) | (qv[3] << 24), qv[4] | (qv[5] << 8) | (qv[6] << 16) | (qv[7] << 24));
        } else {
#pragma unroll
            for (int m = 0; m < 8; ++m)
                if (m < nb) o[m] = (uint8_t)qv[m];
        }
    }
}

}  // namespace

// Returns ZB_ERR_UNSUPPORTED outside its envelope (the caller then runs the two-pass path).
int conv_separable_tile_u8(const zb_image* src, zb_image* dst, int channels, const float* kx, int nx, const float* ky, int ny, int border,
                           cudaStream_t s) {
    if (channels != 1 && channels != 3 && channels != 4) return ZB_ERR_UNSUPPORTED;
    if (images_overlap(src, dst, (size_t)channels)) return ZB_ERR_UNSUPPORTED;     // in place / overlapping views: the temp-plane path
    const int half_x = nx / 2, half_y = ny / 2;
    const int half = half_x > half_y ? half_x : half_y;
    if (half < 1 || half > TU_MAX_HALF) return ZB_ERR_UNSUPPORTED;
    if ((uint64_t)src->cols * channels >= (1u << 30) || src->rows >= (1u << 30)) return ZB_ERR_UNSUPPORTED;
    TileParams p;
    memset(&p, 0, sizeof(p));
    long long sax = 0, say = 0;
    for (int i = 0; i < nx; ++i) {   // Q8 taps, convolution.zig:303-309; tap i acts at offset i - n/2 (:527,542)
        const int q = (int)roundf(kx[i] * 256.0f);
        p.kx[i + (half - half_x)] = q;
        sax += llabs((long long)q);
    }
    for (int i = 0; i < ny; ++i) {
        const int q = (int)roundf(ky[i] * 256.0f);
        p.ky[i + (half - half_y)] = q;
        say += llabs((long long)q);
    }
    if (sax * 255 * say + 32768 >= 2147483647LL) return ZB_ERR_UNSUPPORTED;        // i32 accumulators must be provably safe
    p.src = (const uint8_t*)src->data;
    p.dst = (uint8_t*)dst->data;
    p.src_pitch = (size_t)src->stride * channels;
    p.dst_pitch = (size_t)dst->stride * channels;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.row_bytes = p.cols * channels;
    p.border = border;
    p.src_word_ok = (((uintptr_t)p.src | p.src_pitch | (size_t)p.row_bytes) & 3u) == 0;
    // DP variant: every tap a byte, horizontal sums within 16 bits (the vertical sums then fit 32 bits: 65535 * 255 * 17)
    bool dp = g_tune_u8_dp.load() != 0 && half <= TU_DP_MAX_HALF && sax * 255 <= 65535;
    for (int i = 0; i < 2 * half + 1 && dp; ++i) dp = p.kx[i] >= 0 && p.kx[i] <= 255 && p.ky[i] >= 0 && p.ky[i] <= 255;
    if (dp) {
        const int K = 2 * half + 1;
        for (int m = 0; m < 8; ++m)
            for (int i = 0; i < K; ++i) {
                const int b = m + i * channels;          // byte of the span tap i of output m falls on
                if (b / 4 >= 20) return ZB_ERR_UNSUPPORTED;
                p.tw[m][b / 4] |= (uint32_t)p.kx[i] << (8 * (b % 4));
            }
        for (int q = 0; q <= half; ++q) {
            const int e0 = 2 * q, e1 = 2 * q + 1, o0 = 2 * q - 1, o1 = 2 * q;
            p.kye[q] = (uint32_t)(e0 < K ? p.ky[e0] : 0) | ((uint32_t)(e1 < K ? p.ky[e1] : 0) << 8);
            p.kyo[q] = (uint32_t)(o0 >= 0 ? p.ky[o0] : 0) | ((uint32_t)(o1 < K ? p.ky[o1] : 0) << 8);
        }
        p.dst_word_ok = (((uintptr_t)p.dst | p.dst_pitch) & 3u) == 0;
        p.no_clamp = 255 * sax * say + 32768 < (1LL << 24);
        t_last_kernel = "sep_tile_u8_dp";
        switch (channels) {
            case 1: return launch_half_dp<1>(half, p, s);
            case 3: return launch_half_dp<3>(half, p, s);
            default: return launch_half_dp<4>(half, p, s);
        }
    }
    t_last_kernel = "sep_tile_u8";
    switch (channels) {
        case 1: return launch_half<1>(half, p, s);
        case 3: return launch_half<3>(half, p, s);
        default: return launch_half<4>(half, p, s);
    }
}

// Dense kernels up to 7 x 7 on 8-bit images (`ki`: the kh x kw Q8 taps, row major).  Returns ZB_ERR_UNSUPPORTED outside its envelope
// (the caller then runs the generic kernel).
int convolve_tile_u8(const zb_image* src, zb_image* dst, int channels, const int32_t* ki, int kh, int kw, int border, cudaStream_t s) {
    if (channels != 1 && channels != 3 && channels != 4) return ZB_ERR_UNSUPPORTED;
    if (images_overlap(src, dst, (size_t)channels)) return ZB_ERR_UNSUPPORTED;
    const int half_y = kh / 2, half_x = kw / 2;
    const int half = half_x > half_y ? half_x : half_y;
    if (half < 1 || half > 3) return ZB_ERR_UNSUPPORTED;
    if ((uint64_t)src->cols * channels >= (1u << 30) || src->rows >= (1u << 30)) return ZB_ERR_UNSUPPORTED;
    TileParams p;
    memset(&p, 0, sizeof(p));
    const int K = 2 * half + 1;
    long long sa = 0;
    for (int i = 0; i < kh; ++i)
        for (int j = 0; j < kw; ++j) {   // tap (i, j) acts at offset (i - kh / 2, j - kw / 2) (convolution.zig:216-236)
            p.k2[(i + half - half_y) * K + (j + half - half_x)] = ki[i * kw + j];
            sa += llabs((long long)ki[i * kw + j]);
        }
    if (sa * 255 + 128 >= 2147483647LL) return ZB_ERR_UNSUPPORTED;
    p.src = (const uint8_t*)src->data;
    p.dst = (uint8_t*)dst->data;
    p.src_pitch = (size_t)src->stride * channels;
    p.dst_pitch = (size_t)dst->stride * channels;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.row_bytes = p.cols * channels;
    p.border = border;
    p.src_word_ok = (((uintptr_t)p.src | p.src_pitch | (size_t)p.row_bytes) & 3u) == 0;
    p.dst_dword_ok = (((uintptr_t)p.dst | p.dst_pitch) & 7u) == 0;
    t_last_kernel = "conv2d_tile_u8";
    switch (channels) {
        case 1: return launch_dense_half<1>(half, p, s);
        case 3: return launch_dense_half<3>(half, p, s);
        default: return launch_dense_half<4>(half, p, s);
    }
}

// Image.sobel of an 8-bit image (gray, Rgb, Rgba) into a gray Image(u8) from byte tiles; ZB_ERR_UNSUPPORTED outside its envelope (the
// caller keeps its per-pixel kernel).
int sobel_tile_u8(const zb_image* src, zb_image* dst, int channels, cudaStream_t s) {
    if (channels != 1 && channels != 3 && channels != 4) return ZB_ERR_UNSUPPORTED;
    {   // src and dst have different pixel sizes: compare the byte ranges by hand
        const uintptr_t a0 = (uintptr_t)src->data, a1 = a0 + ((size_t)(src->rows - 1) * src->stride + src->cols) * channels;
        const uintptr_t b0 = (uintptr_t)dst->data, b1 = b0 + ((size_t)(dst->rows - 1) * dst->stride + dst->cols);
        if (a0 < b1 && b0 < a1) return ZB_ERR_UNSUPPORTED;
    }
    if ((uint64_t)src->cols >= (1u << 30) || src->rows >= (1u << 30)) return ZB_ERR_UNSUPPORTED;
    TileParams p;
    memset(&p, 0, sizeof(p));
    p.src = (const uint8_t*)src->data;
    p.dst = (uint8_t*)dst->data;
    p.src_pitch = (size_t)src->stride * channels;
    p.dst_pitch = (size_t)dst->stride;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.row_bytes = p.cols;                      // of the gray tile and of the destination
    p.border = ZB_BORDER_REPLICATE;
    p.src_word_ok = channels == 1 && (((uintptr_t)p.src | p.src_pitch | (size_t)p.row_bytes) & 3u) == 0;
    p.dst_dword_ok = (((uintptr_t)p.dst | p.dst_pitch) & 7u) == 0;
    const dim3 grid = row_grid(div_up((size_t)p.row_bytes, TWB), div_up((size_t)p.rows, 32));
    const int smem = 34 * ((TWB + 2 + 7) & ~7);
    switch (channels) {
        case 1: sobel_tile_u8_kernel<1><<<grid, TWB, smem, s>>>(p); break;
        case 3: sobel_tile_u8_kernel<3><<<grid, TWB, smem, s>>>(p); break;
        default: sobel_tile_u8_kernel<4><<<grid, TWB, smem, s>>>(p); break;
    }
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace zb
