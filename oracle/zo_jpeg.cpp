// zo_jpeg.cpp -- CPU oracle of the baseline JPEG encoder: jpeg.encode (codecs/jpeg.zig:305-325) with encodeRgb (:929-975),
// encodeGrayscale (:977-1042), encodeBlocksRgb (:819-927), encodeBlock (:771-817), fdct8x8_llm (:634-744), quantizeWithRecip
// (:746-768), the segment writers (:452-587) and EntropyWriter (:417-450); the colour conversion is rgbToYcbcr(u8) (color.zig:987-1008).
// TEST INFRASTRUCTURE ONLY (see zignal_oracle.h).  One thread, the reference's loops in the reference's order, i64 where it uses i64.
//
// Only Image(u8) and Image(Rgb(u8)) are encoded here: every other pixel type goes through image.convert(Rgb) first in the reference
// (:319-323), and the binding (tests/jpeg_oracle.py) does that with the main oracle's zo_convert before calling in.
// Built on its own into oracle/libzo_jpeg.so (Makefile).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "zignal_oracle.h"

extern "C" {
int zo_jpeg_encode(const zo_image* src, int pixfmt, int quality, int subsampling, int density_dpi, const uint8_t* comment,
                   int64_t comment_len, uint8_t* out, uint64_t cap, uint64_t* len);
int zo_jpeg_coefficients(const zo_image* src, int pixfmt, int quality, int subsampling, int32_t* coefs, uint64_t cap_blocks,
                         uint64_t* n_blocks);
}

namespace {

constexpr int kUnsupported = 3, kInvalidArgument = 5, kOutOfMemory = 6, kInvalidImageDimensions = 29, kImageTooLarge = 30;

// Zigzag scan order: position i of the scan reads natural index kZigzag[i] (jpeg.zig:49-58, T.81 Figure A.6).
const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// T.81 Annex K, Tables K.1 and K.2 (natural order).
const uint8_t kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,
                            69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
                            81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                              99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                              99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

// Huffman specifications: code-length counts (BITS) and symbols (HUFFVAL).  Both DC tables of the reference are Table K.4's
// (jpeg.zig:356-360); the AC tables are K.5 (luma) and K.6 (chroma).
const uint8_t kDcBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125};
const uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119};
const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// buildHuffmanEncoder (:399-415): canonical codes, shortest first.
struct Huff {
    uint16_t code[256] = {};
    uint8_t size[256] = {};
    Huff(const uint8_t* bits, const uint8_t* vals) {
        uint32_t c = 0;
        int k = 0;
        for (int len = 1; len <= 16; ++len) {
            for (int j = 0; j < bits[len - 1]; ++j, ++k, ++c) {
                code[vals[k]] = (uint16_t)c;
                size[vals[k]] = (uint8_t)len;
            }
            c <<= 1;
        }
    }
};

// EntropyWriter (:417-450): MSB-first bits, 0x00 after every 0xFF byte, flush pads with 1-bits.
struct Bits {
    std::vector<uint8_t>& out;
    uint32_t buf = 0;
    int n = 0;
    void byte(uint8_t b) {
        out.push_back(b);
        if (b == 0xFF) out.push_back(0x00);
    }
    void put(uint32_t v, int size) {
        buf = (buf << size) | (v & ((1u << size) - 1));
        n += size;
        while (n >= 8) {
            byte((uint8_t)(buf >> (n - 8)));
            n -= 8;
        }
    }
    void flush() {
        if (n > 0) {
            const int pad = 8 - n;
            put((1u << pad) - 1, pad);
        }
    }
};

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

// scaleQuantTables (:464-476): libjpeg's quality scaling in integers, clamped to [1, 255].
void scale_tables(int quality, uint8_t* ql, uint8_t* qc) {
    const int q = quality < 1 ? 1 : (quality > 100 ? 100 : quality);
    const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
    for (int i = 0; i < 64; ++i) {
        const int l = (kLumaQ[i] * scale + 50) / 100, c = (kChromaQ[i] * scale + 50) / 100;
        ql[i] = (uint8_t)(l < 1 ? 1 : (l > 255 ? 255 : l));
        qc[i] = (uint8_t)(c < 1 ? 1 : (c > 255 ? 255 : c));
    }
}

// buildQuantRecipLLM (:749-759): round(2^24 / (8 q)) in f64.
void recips(const uint8_t* q, uint32_t* r) {
    for (int i = 0; i < 64; ++i) {
        double f = 16777216.0 / ((double)q[i] * 8.0);
        f = f < 0.0 ? 0.0 : (f > 4294967295.0 ? 4294967295.0 : f);
        r[i] = (uint32_t)__builtin_round(f);
    }
}

// fdct8x8_llm (:634-744), i64 intermediates as in the reference.
constexpr int64_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
                  F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
inline int32_t descale(int64_t x, int n) { return (int32_t)((x + ((int64_t)1 << (n - 1))) >> n); }

void fdct(const int32_t* src, int32_t* dst) {
    int32_t d[64];
    for (int pass = 0; pass < 2; ++pass) {
        const int32_t* in = pass ? d : src;
        int32_t* out = pass ? dst : d;
        const int step = pass ? 8 : 1, lane = pass ? 1 : 8;  // pass 0: rows (elements 1 apart); pass 1: columns (8 apart)
        for (int i = 0; i < 8; ++i) {
            const int32_t* v = in + i * lane;
            int32_t* w = out + i * lane;
            const int64_t t0 = (int64_t)v[0] + v[7 * step], t7 = (int64_t)v[0] - v[7 * step];
            const int64_t t1 = (int64_t)v[step] + v[6 * step], t6 = (int64_t)v[step] - v[6 * step];
            const int64_t t2 = (int64_t)v[2 * step] + v[5 * step], t5 = (int64_t)v[2 * step] - v[5 * step];
            const int64_t t3 = (int64_t)v[3 * step] + v[4 * step], t4 = (int64_t)v[3 * step] - v[4 * step];
            const int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
            if (pass == 0) {
                w[0] = (int32_t)((t10 + t11) << 2);
                w[4 * step] = (int32_t)((t10 - t11) << 2);
            } else {
                w[0] = descale(t10 + t11, 2);
                w[4 * step] = descale(t10 - t11, 2);
            }
            const int sh = pass ? 15 : 11;
            const int64_t z1 = (t12 + t13) * F0541;
            w[2 * step] = descale(z1 + t13 * F0765, sh);
            w[6 * step] = descale(z1 + t12 * -F1847, sh);
            const int64_t z5 = (t4 + t6 + t5 + t7) * F1175;
            const int64_t zo = (t4 + t7) * -F0899, z2 = (t5 + t6) * -F2562;
            const int64_t z3 = (t4 + t6) * -F1961 + z5, z4 = (t5 + t7) * -F0390 + z5;
            w[7 * step] = descale(t4 * F0298 + zo + z3, sh);
            w[5 * step] = descale(t5 * F2053 + z2 + z4, sh);
            w[3 * step] = descale(t6 * F3072 + z2 + z3, sh);
            w[1 * step] = descale(t7 * F1501 + zo + z4, sh);
        }
    }
}

// quantizeWithRecip (:761-768)
inline int32_t quantize(int32_t v, uint32_t recip) {
    if (v == 0) return 0;
    const int64_t a = v < 0 ? -(int64_t)v : v;
    const int64_t q = (a * (int64_t)recip + ((int64_t)1 << 23)) >> 24;
    return (int32_t)(v < 0 ? -q : q);
}

int category(int32_t v) {
    uint32_t a = (uint32_t)(v < 0 ? -v : v);
    int c = 0;
    while (a) { a >>= 1; ++c; }
    return c;
}
uint32_t magnitude_bits(int32_t v, int c) { return c == 0 ? 0 : (v >= 0 ? (uint32_t)v : (uint32_t)(((1 << c) - 1) + v)); }

// The block stage shared by the encoder and the coefficient dump: samples (level-shifted) -> quantised coefficients (natural order).
void block_coefs(const int32_t* samples, const uint32_t* recip, int32_t* q) {
    int32_t dct[64];
    fdct(samples, dct);
    for (int i = 0; i < 64; ++i) q[i] = quantize(dct[i], recip[i]);
}

// encodeBlock (:771-817) after the coefficients: DC difference, then run/size symbols in zigzag order.  A zero run reaching 16 emits
// ZRL at once, trailing zeros included; EOB only when a run is left at the end.
void entropy_block(const int32_t* q, const Huff& dc, const Huff& ac, int32_t* prev_dc, Bits& w) {
    const int32_t diff = q[0] - *prev_dc;
    *prev_dc = q[0];
    const int m = category(diff);
    w.put(dc.code[m], dc.size[m]);
    if (m) w.put(magnitude_bits(diff, m), m);
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int32_t v = q[kZigzag[k]];
        if (v == 0) {
            if (++run == 16) {
                w.put(ac.code[0xF0], ac.size[0xF0]);
                run = 0;
            }
        } else {
            const int c = category(v), sym = (run << 4) | c;
            w.put(ac.code[sym], ac.size[sym]);
            w.put(magnitude_bits(v, c), c);
            run = 0;
        }
    }
    if (run > 0) w.put(ac.code[0x00], ac.size[0x00]);
}

struct Ycc { uint8_t y, cb, cr; };
// rgbToYcbcr(u8) (color.zig:987-1008): 16.16 fixed point, +32768, arithmetic >> 16 on the signed sum, +128 on chroma, clamp.
Ycc to_ycc(const uint8_t* p) {
    const int64_t r = p[0], g = p[1], b = p[2];
    auto clamp = [](int64_t v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); };
    return {clamp((19595 * r + 38470 * g + 7471 * b + 32768) >> 16), clamp(((-11059 * r - 21710 * g + 32768 * b + 32768) >> 16) + 128),
            clamp(((32768 * r - 27439 * g - 5329 * b + 32768) >> 16) + 128)};
}

// Walks the blocks of the image in scan order and hands each one's quantised coefficients and component (0 Y, 1 Cb, 2 Cr) to fn.
// Gray: (:1016-1035).  Colour: encodeBlocksRgb (:819-927), MCU buffer, Y blocks in (vy, hx) order, then Cb, then Cr.
template <typename Fn>
void for_each_block(const zo_image* src, int pixfmt, int subsampling, const uint32_t* rl, const uint32_t* rc, Fn fn) {
    const uint32_t rows = src->rows, cols = src->cols;
    const uint8_t* base = (const uint8_t*)src->data;
    int32_t s[64], q[64];
    if (pixfmt == ZO_PIX_U8) {
        for (uint32_t br = 0; br < (rows + 7) / 8; ++br)
            for (uint32_t bc = 0; bc < (cols + 7) / 8; ++bc) {
                for (int y = 0; y < 8; ++y) {
                    const size_t iy = std::min<size_t>(rows - 1, (size_t)br * 8 + y);
                    for (int x = 0; x < 8; ++x) {
                        const size_t ix = std::min<size_t>(cols - 1, (size_t)bc * 8 + x);
                        s[y * 8 + x] = (int32_t)base[iy * src->stride + ix] - 128;
                    }
                }
                block_coefs(s, rl, q);
                fn(q, 0);
            }
        return;
    }
    const int h = subsampling == 0 ? 1 : 2, v = subsampling == 2 ? 2 : 1;
    const uint32_t mw = 8 * h, mh = 8 * v;
    Ycc mcu[16][16];
    for (uint32_t my = 0; my < (rows + mh - 1) / mh; ++my)
        for (uint32_t mx = 0; mx < (cols + mw - 1) / mw; ++mx) {
            for (uint32_t y = 0; y < mh; ++y) {
                const size_t iy = std::min<size_t>(rows - 1, (size_t)my * mh + y);
                for (uint32_t x = 0; x < mw; ++x) {
                    const size_t ix = std::min<size_t>(cols - 1, (size_t)mx * mw + x);
                    mcu[y][x] = to_ycc(base + (iy * src->stride + ix) * 3);
                }
            }
            for (int vy = 0; vy < v; ++vy)
                for (int hx = 0; hx < h; ++hx) {
                    for (int y = 0; y < 8; ++y)
                        for (int x = 0; x < 8; ++x) s[y * 8 + x] = (int32_t)mcu[vy * 8 + y][hx * 8 + x].y - 128;
                    block_coefs(s, rl, q);
                    fn(q, 0);
                }
            for (int comp = 1; comp <= 2; ++comp) {
                for (int y = 0; y < 8; ++y)
                    for (int x = 0; x < 8; ++x) {
                        uint32_t sum = 0;  // u32 sum, truncating division (:892-899)
                        for (int dy = 0; dy < v; ++dy)
                            for (int dx = 0; dx < h; ++dx) {
                                const Ycc& c = mcu[y * v + dy][x * h + dx];
                                sum += comp == 1 ? c.cb : c.cr;
                            }
                        s[y * 8 + x] = (int32_t)(sum / (uint32_t)(h * v)) - 128;
                    }
                block_coefs(s, rc, q);
                fn(q, comp);
            }
        }
}

int check_args(const zo_image* src, int pixfmt, int subsampling) {
    if (!src) return kInvalidArgument;
    if (pixfmt != ZO_PIX_U8 && pixfmt != ZO_PIX_RGB8) return kUnsupported;
    if (subsampling < 0 || subsampling > 2) return kInvalidArgument;
    if (src->rows == 0 || src->cols == 0) return kInvalidImageDimensions;
    if (src->rows > 65535 || src->cols > 65535) return kImageTooLarge;
    return 0;
}

}  // namespace

extern "C" int zo_jpeg_encode(const zo_image* src, int pixfmt, int quality, int subsampling, int density_dpi, const uint8_t* comment,
                              int64_t comment_len, uint8_t* out, uint64_t cap, uint64_t* len) {
    int rc = check_args(src, pixfmt, subsampling);
    if (rc) return rc;
    if (comment_len > 65533 || !len) return kInvalidArgument;
    const bool gray = pixfmt == ZO_PIX_U8;
    std::vector<uint8_t> o, p;
    o.push_back(0xFF);
    o.push_back(0xD8);
    // APP0 JFIF 1.1, units = dpi (:522-534)
    p = {'J', 'F', 'I', 'F', 0, 1, 1, 1};
    put16(p, density_dpi);
    put16(p, density_dpi);
    p.push_back(0);
    p.push_back(0);
    segment(o, 0xE0, p);
    if (comment_len >= 0) segment(o, 0xFE, std::vector<uint8_t>(comment, comment + comment_len));
    uint8_t ql[64], qc[64];
    scale_tables(quality, ql, qc);
    // DQT in zigzag order (:478-491, :994-998)
    p.clear();
    p.push_back(0x00);
    for (int i = 0; i < 64; ++i) p.push_back(ql[kZigzag[i]]);
    if (!gray) {
        p.push_back(0x01);
        for (int i = 0; i < 64; ++i) p.push_back(qc[kZigzag[i]]);
    }
    segment(o, 0xDB, p);
    // SOF0 (:493-520)
    p = {8};
    put16(p, (int)src->rows);
    put16(p, (int)src->cols);
    if (gray) {
        p.insert(p.end(), {1, 1, 0x11, 0});
    } else {
        const uint8_t yf = subsampling == 0 ? 0x11 : (subsampling == 1 ? 0x21 : 0x22);
        p.insert(p.end(), {3, 1, yf, 0, 2, 0x11, 1, 3, 0x11, 1});
    }
    segment(o, 0xC0, p);
    // DHT (:540-565)
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
    segment(o, 0xC4, p);
    // SOS (:567-587)
    p = gray ? std::vector<uint8_t>{1, 1, 0x00} : std::vector<uint8_t>{3, 1, 0x00, 2, 0x11, 3, 0x11};
    p.insert(p.end(), {0, 63, 0});
    segment(o, 0xDA, p);

    uint32_t rl[64], rcq[64];
    recips(ql, rl);
    recips(qc, rcq);
    const Huff dcl(kDcBits, kDcVals), acl(kAcLumaBits, kAcLumaVals), dcc(kDcBits, kDcVals), acc(kAcChromaBits, kAcChromaVals);
    int32_t prev[3] = {0, 0, 0};
    Bits w{o};
    for_each_block(src, pixfmt, subsampling, rl, rcq, [&](const int32_t* q, int comp) {
        entropy_block(q, comp ? dcc : dcl, comp ? acc : acl, &prev[comp], w);
    });
    w.flush();
    o.push_back(0xFF);
    o.push_back(0xD9);
    *len = o.size();
    if (cap < o.size()) return kOutOfMemory;
    if (out) std::memcpy(out, o.data(), o.size());
    return 0;
}

extern "C" int zo_jpeg_coefficients(const zo_image* src, int pixfmt, int quality, int subsampling, int32_t* coefs, uint64_t cap_blocks,
                                    uint64_t* n_blocks) {
    int rc = check_args(src, pixfmt, subsampling);
    if (rc) return rc;
    uint8_t ql[64], qc[64];
    scale_tables(quality, ql, qc);
    uint32_t rl[64], rcq[64];
    recips(ql, rl);
    recips(qc, rcq);
    uint64_t n = 0;
    for_each_block(src, pixfmt, subsampling, rl, rcq, [&](const int32_t* q, int) {
        if (n < cap_blocks && coefs) std::memcpy(coefs + n * 64, q, 64 * sizeof(int32_t));
        ++n;
    });
    *n_blocks = n;
    return n > cap_blocks ? kOutOfMemory : 0;
}
