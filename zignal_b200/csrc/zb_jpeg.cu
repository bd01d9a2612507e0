// zb_jpeg.cu -- jpeg.encode (codecs/jpeg.zig:305-325): baseline JPEG of a device image, entropy coding included, byte-identical to the
// reference encoder (encodeRgb :929-975, encodeGrayscale :977-1042).
//
// Every 8x8 block is independent up to its DC difference, so the stream is built in parallel:
//   1. jpeg_blocks   one CTA per group of MCUs: load the MCU with the edge rule (@min(rows-1, .), :863-866), convert the pixel to Rgb(u8)
//                    (convert_color, as image.convert(Rgb) does for the other pixel types, :319-323), rgbToYcbcr (color.zig:987-1008),
//                    the truncating chroma average (:884-923), the LLM FDCT (:634-744) with 8 threads per block (a row each, then a
//                    column each), reciprocal quantisation (:749-768).  Writes each block's 64 quantised coefficients in zigzag order
//                    (i16), its DC, and the bit count of its AC symbols, which depends on the block alone.
//   2. jpeg_bits     each block's total bit count: the AC count plus the DC code of the difference to the previous block of the same
//                    component in scan order (one predictor per component, no restart intervals).
//   3. scan          exclusive prefix sum of the bit counts into 64-bit bit offsets (per-tile partials, one CTA over the partials,
//                    then the tiles again).  The total comes back to the host to size the stream.
//   4. jpeg_emit     each block writes its codes at its bit offset into a zeroed buffer of big-endian 32-bit words: the two words it
//                    may share with its neighbours through atomicOr, the words in between with plain stores.  The last block appends
//                    the 1-bit padding of EntropyWriter.flush (:444-449).
//   5. jpeg_stuff    0xFF bytes are counted per 16-byte chunk, the counts are scanned, and every byte is scattered to its final place
//                    with a 0x00 after each 0xFF (:430-433).  The stuffed length comes back to the host, and after the capacity check
//                    the bytes follow.
// The header (about 600 bytes) is written on the host straight into the caller's buffer, followed by the entropy segment and EOI.
//
// Scratch, all stream-ordered: 148 bytes per block (128 coefficients, 4 DC, 4 AC bits, 4 total bits, 8 offset), the packed stream
// rounded up to 16 bytes, 4 + 8 bytes per 16 stream bytes for the stuffing counts and offsets, and the stuffed stream.
//
// The FDCT runs in i32 where the reference uses i64: with samples in [-128, 127] every intermediate of both passes stays below
// 3.2e8 < 2^31 / 6 (tests/test_jpeg_host.py propagates the intervals), so both give the same bits.  The quantisation product needs 64 bits.
#include <cstring>
#include <vector>

#include "zb_convert.cuh"
#include "zb_jpeg_common.cuh"
#include "zb_internal.h"

namespace zb {
namespace {


// T.81 Annex K, Tables K.1 (luminance) and K.2 (chrominance), natural order (jpeg.zig:333-352).
constexpr uint8_t kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,
                                69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
                                81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                  99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

// Huffman specifications (jpeg.zig:354-391): BITS (codes per length 1..16) and HUFFVAL.  Both DC tables are Table K.4's, which has
// the category 11 that a DC difference reaches when the DC divisor is 1 (quality >= 96); the AC tables are K.5 and K.6.
constexpr uint8_t kDcBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125};
constexpr uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
constexpr uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119};
constexpr uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// Code and length of every symbol of the four tables (buildHuffmanEncoder, :399-415): [0] DC luma, [1] AC luma, [2] DC chroma,
// [3] AC chroma.
struct HuffTables {
    uint16_t code[4][256];
    uint8_t size[4][256];
};
constexpr void canonical(HuffTables& t, int id, const uint8_t* bits, const uint8_t* vals) {
    uint32_t c = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int j = 0; j < bits[len - 1]; ++j, ++k, ++c) {
            t.code[id][vals[k]] = (uint16_t)c;
            t.size[id][vals[k]] = (uint8_t)len;
        }
        c <<= 1;
    }
}
constexpr HuffTables make_tables() {
    HuffTables t{};
    canonical(t, 0, kDcBits, kDcVals);
    canonical(t, 1, kAcLumaBits, kAcLumaVals);
    canonical(t, 2, kDcBits, kDcVals);
    canonical(t, 3, kAcChromaBits, kAcChromaVals);
    return t;
}
__constant__ HuffTables c_huff = make_tables();

// Natural index -> zigzag scan position.
constexpr uint8_t inverse_zigzag(int n) {
    for (int i = 0; i < 64; ++i)
        if (kZigzag[i] == n) return (uint8_t)i;
    return 0;
}
struct InvZigzag { uint8_t v[64]; };
constexpr InvZigzag make_inv_zigzag() {
    InvZigzag z{};
    for (int n = 0; n < 64; ++n) z.v[n] = inverse_zigzag(n);
    return z;
}
__constant__ InvZigzag c_unzig = make_inv_zigzag();

// Reciprocal divisors round(2^24 / (8 q)) of the luma [0] and chroma [1] tables (buildQuantRecipLLM, :749-759).
struct Recips { uint32_t r[2][64]; };

constexpr int kBlocksPerCta = 32;       // jpeg_blocks: 8 threads per block
constexpr int kBlockThreads = kBlocksPerCta * 8;
constexpr int kStuffChunk = 16;         // bytes per thread of the stuffing pass
constexpr int kMaxBlockBits = 22 + 63 * 26;   // DC: 11-bit code + 11 magnitude bits; AC: 16-bit code + 10 magnitude bits
constexpr int kZrl = 0xF0, kEob = 0x00;

__device__ __forceinline__ int category(int v) { return v == 0 ? 0 : 32 - __clz(v < 0 ? -v : v); }
__device__ __forceinline__ uint32_t magnitude_bits(int v, int c) { return v >= 0 ? (uint32_t)v : (uint32_t)(v + (1 << c) - 1); }

// One pass of fdct8x8_llm over 8 values; PASS 0 (rows) scales by 2^2, PASS 1 (columns) removes that again (:643-743).
template <int PASS>
__device__ __forceinline__ void fdct8(const int* v, int* o) {
    constexpr int C0298 = 2446, C0390 = 3196, C0541 = 4433, C0765 = 6270, C0899 = 7373, C1175 = 9633, C1501 = 12299, C1847 = 15137,
                  C1961 = 16069, C2053 = 16819, C2562 = 20995, C3072 = 25172;
    constexpr int SH = PASS == 0 ? 11 : 15;
    auto descale = [](int x, int n) { return (x + (1 << (n - 1))) >> n; };
    const int t0 = v[0] + v[7], t7 = v[0] - v[7], t1 = v[1] + v[6], t6 = v[1] - v[6];
    const int t2 = v[2] + v[5], t5 = v[2] - v[5], t3 = v[3] + v[4], t4 = v[3] - v[4];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    if (PASS == 0) {
        o[0] = (t10 + t11) * 4;
        o[4] = (t10 - t11) * 4;
    } else {
        o[0] = descale(t10 + t11, 2);
        o[4] = descale(t10 - t11, 2);
    }
    const int z1 = (t12 + t13) * C0541;
    o[2] = descale(z1 + t13 * C0765, SH);
    o[6] = descale(z1 - t12 * C1847, SH);
    const int z5 = (t4 + t6 + t5 + t7) * C1175;
    const int zo = -(t4 + t7) * C0899, z2 = -(t5 + t6) * C2562;
    const int z3 = z5 - (t4 + t6) * C1961, z4 = z5 - (t5 + t7) * C0390;
    o[7] = descale(t4 * C0298 + zo + z3, SH);
    o[5] = descale(t5 * C2053 + z2 + z4, SH);
    o[3] = descale(t6 * C3072 + z2 + z3, SH);
    o[1] = descale(t7 * C1501 + zo + z4, SH);
}

// quantizeWithRecip (:761-768)
__device__ __forceinline__ int quantize(int v, uint32_t recip) {
    const long long a = v < 0 ? -(long long)v : v;
    const int q = (int)((a * recip + (1ll << 23)) >> 24);
    return v < 0 ? -q : q;
}

// rgbToYcbcr(u8) (color.zig:987-1008): 16.16 fixed point rounded at +32768, arithmetic >> 16 of the signed sum, +128, clamp.
__device__ __forceinline__ void to_ycc(int r, int g, int b, uint8_t& y, uint8_t& cb, uint8_t& cr) {
    y = (uint8_t)min(max((19595 * r + 38470 * g + 7471 * b + 32768) >> 16, 0), 255);
    cb = (uint8_t)min(max(((-11059 * r - 21710 * g + 32768 * b + 32768) >> 16) + 128, 0), 255);
    cr = (uint8_t)min(max(((32768 * r - 27439 * g - 5329 * b + 32768) >> 16) + 128, 0), 255);
}

// Blocks per MCU and MCU geometry of a layout: SUB -1 = grayscale, 0 / 1 / 2 = 4:4:4 / 4:2:2 / 4:2:0 colour (:832-843).
template <int SUB> struct Layout {
    static constexpr int H = SUB <= 0 ? 1 : 2, V = SUB == 2 ? 2 : 1;
    static constexpr int LUMA = H * V, PER_MCU = SUB < 0 ? 1 : LUMA + 2;
    static constexpr int MW = 8 * H, MH = 8 * V;
    static constexpr int MCUS = kBlocksPerCta / PER_MCU;   // MCUs per CTA of jpeg_blocks
};

struct Geometry {
    uint32_t rows, cols;
    uint32_t mcu_cols;
    uint64_t mcus, blocks;
};

// Stage 1.  coef: 64 i16 per block in zigzag order; dc: the quantised DC; acbits: the bits of the block's AC symbols.
template <int SF, int SUB>
__global__ void __launch_bounds__(kBlockThreads) jpeg_blocks(const uint8_t* __restrict__ src, uint64_t stride, Geometry g, Recips q,
                                                             int16_t* __restrict__ coef, int* __restrict__ dc, uint32_t* __restrict__ acbits) {
    using L = Layout<SUB>;
    using CT = typename Fmt<SF>::CT;
    constexpr int PB = (int)sizeof(CT) * Fmt<SF>::N;
    constexpr int PLANES = SUB < 0 ? 1 : 3;
    __shared__ uint8_t pix[PLANES][L::MCUS][L::MH][L::MW];
    __shared__ int rowpass[kBlocksPerCta][64];
    __shared__ __align__(16) int16_t zz[kBlocksPerCta][64];

    const uint64_t mcu0 = (uint64_t)blockIdx.x * L::MCUS;
    const int nmcu = (int)min((uint64_t)L::MCUS, g.mcus - mcu0);
    const int nblk = nmcu * L::PER_MCU;

    // MCU buffer: the replicated edge, converted once per pixel
    for (int i = threadIdx.x; i < nmcu * L::MH * L::MW; i += blockDim.x) {
        const int m = i / (L::MH * L::MW), y = (i / L::MW) % L::MH, x = i % L::MW;
        const uint64_t mcu = mcu0 + m;
        const uint32_t my = (uint32_t)(mcu / g.mcu_cols), mx = (uint32_t)(mcu % g.mcu_cols);
        const uint32_t iy = min(g.rows - 1, my * L::MH + y), ix = min(g.cols - 1, mx * L::MW + x);
        const CT* p = (const CT*)(src + ((uint64_t)iy * stride + ix) * PB);
        if constexpr (SUB < 0) {
            pix[0][m][y][x] = p[0];
        } else {
            uint8_t rgb[3];
            if constexpr (SF == ZB_PIX_RGB8) {
                rgb[0] = p[0]; rgb[1] = p[1]; rgb[2] = p[2];
            } else {
                CT s[Fmt<SF>::N];
#pragma unroll
                for (int k = 0; k < Fmt<SF>::N; ++k) s[k] = p[k];
                convert_color<SF, ZB_PIX_RGB8>(s, rgb);
            }
            to_ycc(rgb[0], rgb[1], rgb[2], pix[0][m][y][x], pix[1][m][y][x], pix[2][m][y][x]);
        }
    }
    __syncthreads();

    // Samples of row r of block j, level-shifted, then the row pass
    const int j = threadIdx.x >> 3, r = threadIdx.x & 7;
    const bool live = j < nblk;
    const int m = j / L::PER_MCU, k = j % L::PER_MCU;
    const int comp = k < L::LUMA ? 0 : k - L::LUMA + 1;
    if (live) {
        int s[8], o[8];
        if (comp == 0) {
            const int vy = k / L::H, hx = k % L::H;
#pragma unroll
            for (int x = 0; x < 8; ++x) s[x] = (int)pix[0][m][vy * 8 + r][hx * 8 + x] - 128;
        } else {
#pragma unroll
            for (int x = 0; x < 8; ++x) {
                uint32_t sum = 0;
#pragma unroll
                for (int dy = 0; dy < L::V; ++dy)
#pragma unroll
                    for (int dx = 0; dx < L::H; ++dx) sum += pix[comp][m][r * L::V + dy][x * L::H + dx];
                s[x] = (int)(sum / (uint32_t)L::LUMA) - 128;
            }
        }
        fdct8<0>(s, o);
#pragma unroll
        for (int u = 0; u < 8; ++u) rowpass[j][r * 8 + u] = o[u];
    }
    __syncthreads();

    // Column pass (thread r takes column r) and quantisation into zigzag order
    if (live) {
        int s[8], o[8];
#pragma unroll
        for (int v = 0; v < 8; ++v) s[v] = rowpass[j][v * 8 + r];
        fdct8<1>(s, o);
        const uint32_t* rc = q.r[comp ? 1 : 0];
#pragma unroll
        for (int u = 0; u < 8; ++u) zz[j][c_unzig.v[u * 8 + r]] = (int16_t)quantize(o[u], rc[u * 8 + r]);
    }
    __syncthreads();

    // AC bits: the 8 threads of a block each take 8 scan positions; the nonzero mask of the whole block comes from the 8 lanes.
    uint64_t mine = 0;
    if (live) {
#pragma unroll
        for (int i = 0; i < 8; ++i) mine |= (uint64_t)(zz[j][r * 8 + i] != 0) << (r * 8 + i);
    }
    mine &= ~1ull;   // the DC
    uint64_t mask = mine;
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) mask |= __shfl_xor_sync(0xffffffffu, mask, d);
    const int tab = comp ? 3 : 1;
    const int zrl = c_huff.size[tab][kZrl];
    uint32_t bits = 0;
    for (uint64_t w = mine; w; w &= w - 1) {
        const int p = __ffsll((long long)w) - 1;
        const uint64_t below = mask & ((1ull << p) - 1);
        const int prev = below ? 63 - __clzll((long long)below) : 0;
        const int run = p - prev - 1, c = category(zz[j][p]);
        bits += (run >> 4) * zrl + c_huff.size[tab][((run & 15) << 4) | c] + c;
    }
    if (r == 7) {   // trailing zeros: a ZRL per 16, EOB for a remainder
        const int last = mask ? 63 - __clzll((long long)mask) : 0, t = 63 - last;
        bits += (t >> 4) * zrl + ((t & 15) ? c_huff.size[tab][kEob] : 0);
    }
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) bits += __shfl_xor_sync(0xffffffffu, bits, d);
    const uint64_t b0 = mcu0 * L::PER_MCU;
    if (live && r == 0) {
        dc[b0 + j] = zz[j][0];
        acbits[b0 + j] = bits;
    }
    // coefficients out, 16 bytes per thread
    const uint4* from = (const uint4*)&zz[0][0];
    uint4* to = (uint4*)(coef + b0 * 64);
    for (int i = threadIdx.x; i < nblk * 8; i += blockDim.x) to[i] = from[i];
}

// Block b of the scan: component (0 Y, 1 Cb, 2 Cr) and the block that holds its DC predictor (-1: none, the predictor is 0).
__device__ __forceinline__ void block_role(uint64_t b, int per_mcu, int luma, int& comp, int64_t& pred) {
    if (per_mcu == 1) {
        comp = 0;
        pred = (int64_t)b - 1;
        return;
    }
    const int k = (int)(b % per_mcu);
    comp = k < luma ? 0 : k - luma + 1;
    if (comp == 0 && k > 0) pred = (int64_t)b - 1;
    else pred = b >= (uint64_t)per_mcu ? (int64_t)(b - per_mcu + (comp == 0 ? luma - 1 : 0)) : -1;
}

// Stage 2: the bits of block b.
__global__ void __launch_bounds__(kThreads) jpeg_bits(const int* __restrict__ dc, const uint32_t* __restrict__ acbits, uint64_t n,
                                                      int per_mcu, int luma, uint32_t* __restrict__ len) {
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    int comp;
    int64_t pred;
    block_role(b, per_mcu, luma, comp, pred);
    const int c = category(dc[b] - (pred >= 0 ? dc[pred] : 0));
    len[b] = acbits[b] + c_huff.size[comp ? 2 : 0][c] + c;
}

// Big-endian word writer: bits are appended MSB first from bit offset `pos` of a zeroed buffer of 32-bit words.
struct BitSink {
    uint32_t* words;
    uint64_t w;        // index of the word being filled
    uint64_t acc;      // pending bits, the last `n` of them valid
    int n;             // bits of word w held in acc (counting the ones before pos that belong to the previous block as zeros)
    bool first;        // word w may hold bits of the previous block
    __device__ BitSink(uint32_t* words_, uint64_t pos) : words(words_), w(pos >> 5), acc(0), n((int)(pos & 31)), first(true) {}
    __device__ __forceinline__ void store(uint32_t v, bool shared) {
        const uint32_t be = __byte_perm(v, 0, 0x0123);
        if (shared) atomicOr(words + w, be);
        else words[w] = be;
    }
    __device__ __forceinline__ void put(uint32_t v, int len) {   // len <= 26
        acc = (acc << len) | v;
        n += len;
        if (n >= 32) {
            n -= 32;
            store((uint32_t)(acc >> n), first);
            first = false;
            ++w;
        }
    }
    __device__ __forceinline__ void finish() {   // the last word is shared with the next block
        if (n > 0) store((uint32_t)(acc << (32 - n)), true);
    }
};

// Stage 4: the codes of block b at bit offset off[b] (encodeBlock's symbols, :786-816).
__global__ void __launch_bounds__(kThreads) jpeg_emit(const int16_t* __restrict__ coef, const int* __restrict__ dc,
                                                      const uint64_t* __restrict__ off, uint64_t n, int per_mcu, int luma,
                                                      uint32_t* __restrict__ words) {
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    int comp;
    int64_t pred;
    block_role(b, per_mcu, luma, comp, pred);
    const int dtab = comp ? 2 : 0, atab = comp ? 3 : 1;
    const int16_t* cz = coef + b * 64;
    uint64_t mask = 0;
    const uint4* c4 = (const uint4*)cz;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint4 u = c4[i];
        const uint32_t h[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            mask |= (uint64_t)((h[k] & 0xFFFFu) != 0) << (i * 8 + k * 2);
            mask |= (uint64_t)((h[k] >> 16) != 0) << (i * 8 + k * 2 + 1);
        }
    }
    mask &= ~1ull;
    BitSink out(words, off[b]);
    const int diff = dc[b] - (pred >= 0 ? dc[pred] : 0), dcat = category(diff);
    out.put(((uint32_t)c_huff.code[dtab][dcat] << dcat) | (dcat ? magnitude_bits(diff, dcat) : 0), c_huff.size[dtab][dcat] + dcat);
    const uint32_t zrl_code = c_huff.code[atab][kZrl];
    const int zrl_size = c_huff.size[atab][kZrl];
    int prev = 0;
    for (uint64_t w = mask; w; w &= w - 1) {
        const int p = __ffsll((long long)w) - 1;
        int run = p - prev - 1;
        for (; run >= 16; run -= 16) out.put(zrl_code, zrl_size);
        const int v = cz[p], c = category(v), sym = (run << 4) | c;
        out.put(((uint32_t)c_huff.code[atab][sym] << c) | magnitude_bits(v, c), c_huff.size[atab][sym] + c);
        prev = p;
    }
    int t = 63 - prev;
    for (; t >= 16; t -= 16) out.put(zrl_code, zrl_size);
    if (t) out.put(c_huff.code[atab][kEob], c_huff.size[atab][kEob]);
    if (b == n - 1) {   // EntropyWriter.flush: pad the last byte with 1-bits
        const int used = out.n & 7;
        if (used) out.put((1u << (8 - used)) - 1, 8 - used);
    }
    out.finish();
}

// Stage 5a: 0xFF bytes of each 16-byte chunk of the packed stream.
__global__ void __launch_bounds__(kThreads) jpeg_count_ff(const uint4* __restrict__ stream, uint64_t chunks, uint32_t* __restrict__ cnt) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= chunks) return;
    const uint4 u = stream[t];
    const uint32_t h[4] = {u.x, u.y, u.z, u.w};
    uint32_t c = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) c += __popc(__vcmpeq4(h[k], 0xFFFFFFFFu)) / 8;
    cnt[t] = c;   // bytes past the stream's end are zero, never 0xFF
}

// Stage 5b: every byte to its place, a 0x00 after each 0xFF.
__global__ void __launch_bounds__(kThreads) jpeg_stuff(const uint4* __restrict__ stream, uint64_t nbytes, const uint64_t* __restrict__ ffs,
                                                       uint8_t* __restrict__ out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t first = t * kStuffChunk;
    if (first >= nbytes) return;
    const uint4 u = stream[t];
    const uint32_t h[4] = {u.x, u.y, u.z, u.w};
    uint64_t pos = first + ffs[t];
    const int cnt = (int)min((uint64_t)kStuffChunk, nbytes - first);
#pragma unroll
    for (int i = 0; i < kStuffChunk; ++i) {
        if (i < cnt) {
            const uint8_t v = (uint8_t)(h[i >> 2] >> ((i & 3) * 8));
            out[pos++] = v;
            if (v == 0xFF) out[pos++] = 0x00;
        }
    }
}

// ---- host side --------------------------------------------------------------------------------------------------------------------

int subsampling_of(int pixfmt, int subsampling) { return pixfmt == ZB_PIX_U8 ? -1 : subsampling; }

void quant_tables(int quality, uint8_t* ql, uint8_t* qc) {   // scaleQuantTables (:464-476)
    const int q = quality < 1 ? 1 : (quality > 100 ? 100 : quality);
    const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
    for (int i = 0; i < 64; ++i) {
        const int l = (kLumaQ[i] * scale + 50) / 100, c = (kChromaQ[i] * scale + 50) / 100;
        ql[i] = (uint8_t)(l < 1 ? 1 : (l > 255 ? 255 : l));
        qc[i] = (uint8_t)(c < 1 ? 1 : (c > 255 ? 255 : c));
    }
}

void put16(std::vector<uint8_t>& o, int v) {
    o.push_back((uint8_t)(v >> 8));
    o.push_back((uint8_t)v);
}
void segment(std::vector<uint8_t>& o, uint8_t marker, const std::vector<uint8_t>& payload) {
    o.push_back(0xFF);
    o.push_back(marker);
    put16(o, (int)payload.size() + 2);
    o.insert(o.end(), payload.begin(), payload.end());
}

// SOI, APP0 (JFIF 1.1, dpi), COM, DQT, SOF0, DHT, SOS: the writers of :452-587 in encodeRgb's / encodeGrayscale's order.
std::vector<uint8_t> header(uint32_t rows, uint32_t cols, int sub, const zb_jpeg_options& o) {
    const bool gray = sub < 0;
    std::vector<uint8_t> h = {0xFF, 0xD8}, p = {'J', 'F', 'I', 'F', 0, 1, 1, 1};
    put16(p, o.density_dpi);
    put16(p, o.density_dpi);
    p.push_back(0);
    p.push_back(0);
    segment(h, 0xE0, p);
    if (o.comment) segment(h, 0xFE, std::vector<uint8_t>(o.comment, o.comment + o.comment_len));
    uint8_t ql[64], qc[64];
    quant_tables(o.quality, ql, qc);
    p = {0x00};
    for (int i = 0; i < 64; ++i) p.push_back(ql[kZigzag[i]]);
    if (!gray) {
        p.push_back(0x01);
        for (int i = 0; i < 64; ++i) p.push_back(qc[kZigzag[i]]);
    }
    segment(h, 0xDB, p);
    p = {8};
    put16(p, (int)rows);
    put16(p, (int)cols);
    if (gray) p.insert(p.end(), {1, 1, 0x11, 0});
    else p.insert(p.end(), {3, 1, (uint8_t)(sub == 0 ? 0x11 : (sub == 1 ? 0x21 : 0x22)), 0, 2, 0x11, 1, 3, 0x11, 1});
    segment(h, 0xC0, p);
    p.clear();
    auto table = [&p](uint8_t tc, const uint8_t* bits, const uint8_t* vals, int nv) {
        p.push_back(tc);
        p.insert(p.end(), bits, bits + 16);
        p.insert(p.end(), vals, vals + nv);
    };
    table(0x00, kDcBits, kDcVals, 12);
    table(0x10, kAcLumaBits, kAcLumaVals, 162);
    if (!gray) {
        table(0x01, kDcBits, kDcVals, 12);
        table(0x11, kAcChromaBits, kAcChromaVals, 162);
    }
    segment(h, 0xC4, p);
    p = gray ? std::vector<uint8_t>{1, 1, 0x00} : std::vector<uint8_t>{3, 1, 0x00, 2, 0x11, 3, 0x11};
    p.insert(p.end(), {0, 63, 0});
    segment(h, 0xDA, p);
    return h;
}

Geometry geometry(uint32_t rows, uint32_t cols, int sub) {
    const int h = sub <= 0 ? 1 : 2, v = sub == 2 ? 2 : 1, per = sub < 0 ? 1 : h * v + 2;
    Geometry g;
    g.rows = rows;
    g.cols = cols;
    g.mcu_cols = (cols + 8 * h - 1) / (8 * h);
    g.mcus = (uint64_t)((rows + 8 * v - 1) / (8 * v)) * g.mcu_cols;
    g.blocks = g.mcus * per;
    return g;
}

int check_args(uint32_t rows, uint32_t cols, int pixfmt, const zb_jpeg_options* o) {
    if (!o) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if (rows == 0 || cols == 0) return ZB_ERR_INVALID_IMAGE_DIMENSIONS;   // :309-314
    if (rows > 65535 || cols > 65535) return ZB_ERR_IMAGE_TOO_LARGE;
    if (o->subsampling > ZB_JPEG_YUV420) return ZB_ERR_INVALID_ARGUMENT;
    if (o->comment && o->comment_len > 65533) return ZB_ERR_INVALID_ARGUMENT;   // the segment length is a u16 counting itself
    return ZB_OK;
}

template <int SF, int SUB>
void launch_blocks(const zb_image* src, const Geometry& g, const Recips& q, int16_t* coef, int* dc, uint32_t* acbits, cudaStream_t s) {
    const uint64_t ctas = (g.mcus + Layout<SUB>::MCUS - 1) / Layout<SUB>::MCUS;
    jpeg_blocks<SF, SUB><<<(unsigned)ctas, kBlockThreads, 0, s>>>((const uint8_t*)src->data, src->stride, g, q, coef, dc, acbits);
}

template <int SF>
void launch_colour(int sub, const zb_image* src, const Geometry& g, const Recips& q, int16_t* coef, int* dc, uint32_t* acbits,
                   cudaStream_t s) {
    if (sub == 0) launch_blocks<SF, 0>(src, g, q, coef, dc, acbits, s);
    else if (sub == 1) launch_blocks<SF, 1>(src, g, q, coef, dc, acbits, s);
    else launch_blocks<SF, 2>(src, g, q, coef, dc, acbits, s);
}

const char* kernel_name(int pixfmt, int sub) {
    static const char* names[5][3] = {{"jpeg_gray_u8", "jpeg_gray_u8", "jpeg_gray_u8"},
                                      {"jpeg_444_f32", "jpeg_422_f32", "jpeg_420_f32"},
                                      {"jpeg_444_rgb8", "jpeg_422_rgb8", "jpeg_420_rgb8"},
                                      {"jpeg_444_rgba8", "jpeg_422_rgba8", "jpeg_420_rgba8"},
                                      {"jpeg_444_rgbaf32", "jpeg_422_rgbaf32", "jpeg_420_rgbaf32"}};
    return names[pixfmt][sub < 0 ? 0 : sub];
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_jpeg_encode_bound(uint32_t rows, uint32_t cols, int pixfmt, const zb_jpeg_options* opts, uint64_t* bytes) {
    if (!bytes) return ZB_ERR_INVALID_ARGUMENT;
    const int rc = check_args(rows, cols, pixfmt, opts);
    if (rc) return rc;
    const int sub = subsampling_of(pixfmt, opts->subsampling);
    const Geometry g = geometry(rows, cols, sub);
    // every block at its longest, in whole bytes (which also covers the padded last byte), doubled for stuffing; header and EOI
    *bytes = header(rows, cols, sub, *opts).size() + g.blocks * 2 * ((kMaxBlockBits + 7) / 8) + 2;
    return ZB_OK;
}

extern "C" int zb_jpeg_encode(const zb_image* src, int pixfmt, const zb_jpeg_options* opts, uint8_t* out_host, uint64_t cap, uint64_t* len,
                              zb_stream stream) {
    if (!src || !len) return ZB_ERR_INVALID_ARGUMENT;
    int rc = check_args(src->rows, src->cols, pixfmt, opts);
    if (rc) return rc;
    if (!src->data || src->stride < src->cols || (!out_host && cap > 0)) return ZB_ERR_INVALID_ARGUMENT;
    cudaStream_t s = (cudaStream_t)stream;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;

    const int sub = subsampling_of(pixfmt, opts->subsampling);
    const Geometry g = geometry(src->rows, src->cols, sub);
    const std::vector<uint8_t> head = header(src->rows, src->cols, sub, *opts);
    uint8_t ql[64], qc[64];
    quant_tables(opts->quality, ql, qc);
    Recips q;
    for (int i = 0; i < 64; ++i) {   // buildQuantRecipLLM: round(2^24 / (8 q)) in f64
        q.r[0][i] = (uint32_t)__builtin_round(16777216.0 / ((double)ql[i] * 8.0));
        q.r[1][i] = (uint32_t)__builtin_round(16777216.0 / ((double)qc[i] * 8.0));
    }
    const int per_mcu = sub < 0 ? 1 : (sub == 0 ? 1 : 2) * (sub == 2 ? 2 : 1) + 2, luma = sub < 0 ? 1 : per_mcu - 2;

    // per-block scratch: coefficients, DC, AC bits (reused for the total bits), offsets (+1 for the total), scan partials
    const uint64_t n = g.blocks, tiles = (n + kScanTile - 1) / kScanTile;
    Scratch blk;
    const size_t coef_b = n * 128, dc_b = n * 4, bits_b = n * 4, off_b = (n + 1) * 8, part_b = tiles * 8;
    if ((rc = blk.alloc(coef_b + dc_b + 2 * bits_b + off_b + part_b + 64, s))) return rc;
    int16_t* coef = blk.as<int16_t>();
    int* dc = (int*)((char*)blk.p + coef_b);
    uint32_t* acbits = (uint32_t*)((char*)dc + dc_b);
    uint32_t* bits = acbits + n;
    uint64_t* off = (uint64_t*)(((uintptr_t)(bits + n) + 15) & ~(uintptr_t)15);
    uint64_t* part = off + n + 1;

    switch (pixfmt) {
        case ZB_PIX_U8: launch_blocks<ZB_PIX_U8, -1>(src, g, q, coef, dc, acbits, s); break;
        case ZB_PIX_F32: launch_colour<ZB_PIX_F32>(sub, src, g, q, coef, dc, acbits, s); break;
        case ZB_PIX_RGB8: launch_colour<ZB_PIX_RGB8>(sub, src, g, q, coef, dc, acbits, s); break;
        case ZB_PIX_RGBA8: launch_colour<ZB_PIX_RGBA8>(sub, src, g, q, coef, dc, acbits, s); break;
        default: launch_colour<ZB_PIX_RGBAF32>(sub, src, g, q, coef, dc, acbits, s); break;
    }
    ZB_LAUNCHED();
    jpeg_bits<<<div_up(n, kThreads), kThreads, 0, s>>>(dc, acbits, n, per_mcu, luma, bits);
    ZB_LAUNCHED();
    if ((rc = scan(bits, n, part, off, s))) return rc;
    uint64_t total_bits = 0;
    ZB_CUDA(cudaMemcpyAsync(&total_bits, off + n, 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));

    // the packed stream, whole 16-byte chunks, zeroed
    const uint64_t nbytes = (total_bits + 7) / 8, chunks = (nbytes + kStuffChunk - 1) / kStuffChunk;
    Scratch st;
    if ((rc = st.alloc(chunks * kStuffChunk + chunks * 4 + (chunks + 1) * 8 + ((chunks + kScanTile - 1) / kScanTile) * 8 + 64, s)))
        return rc;
    uint32_t* words = st.as<uint32_t>();
    uint32_t* cnt = (uint32_t*)((char*)st.p + chunks * kStuffChunk);
    uint64_t* ffs = (uint64_t*)(((uintptr_t)(cnt + chunks) + 15) & ~(uintptr_t)15);
    uint64_t* part2 = ffs + chunks + 1;
    ZB_CUDA(cudaMemsetAsync(words, 0, chunks * kStuffChunk, s));
    jpeg_emit<<<div_up(n, kThreads), kThreads, 0, s>>>(coef, dc, off, n, per_mcu, luma, words);
    ZB_LAUNCHED();
    jpeg_count_ff<<<div_up(chunks, kThreads), kThreads, 0, s>>>((const uint4*)words, chunks, cnt);
    ZB_LAUNCHED();
    if ((rc = scan(cnt, chunks, part2, ffs, s))) return rc;
    uint64_t n_ff = 0;
    ZB_CUDA(cudaMemcpyAsync(&n_ff, ffs + chunks, 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));

    const uint64_t body = nbytes + n_ff;
    *len = head.size() + body + 2;
    t_last_kernel = kernel_name(pixfmt, sub);
    if (cap < *len) return ZB_ERR_OUT_OF_MEMORY;
    Scratch stuffed;
    if ((rc = stuffed.alloc(body, s))) return rc;
    jpeg_stuff<<<div_up(chunks, kThreads), kThreads, 0, s>>>((const uint4*)words, nbytes, ffs, stuffed.as<uint8_t>());
    ZB_LAUNCHED();
    ZB_CUDA(cudaMemcpyAsync(out_host + head.size(), stuffed.p, body, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    std::memcpy(out_host, head.data(), head.size());
    out_host[head.size() + body] = 0xFF;
    out_host[head.size() + body + 1] = 0xD9;
    return ZB_OK;
}
