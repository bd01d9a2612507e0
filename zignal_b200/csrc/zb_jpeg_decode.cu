// zb_jpeg_decode.cu -- jpeg.loadFromBytes (codecs/jpeg.zig:2825-2851) for baseline streams: the file's bytes go to the device once and
// the whole entropy-coded segment is decoded there, in parallel, into a caller-allocated device image of any pixel format.
//
// The host parses the segments before the first SOS as decode does (:2035-2157, parseSOF / DHT / DQT / SOS / DRI :1311-1644), builds the
// decode tables, and copies the bytes after the SOS header to the device in one transfer.  It never reads the entropy-coded bytes.
// The device then runs:
//   1. dec_scan_end     findScanEnd (:1955-1978) as a parallel min over the terminating FF positions.
//   2. dec_destuff_*    count / scan / scatter: the 00 after each FF and every RST marker are removed (the inverse of the encoder's
//                       jpeg_count_ff / jpeg_stuff), and each RST's destuffed offset is recorded as the start of a restart interval.
//   3. dec_subs         the destuffed stream is cut into subsequences of kSubBits bits, never across an interval start.
//   4. dec_sync         self-synchronising Huffman decoding (Weissenberger & Schmidt, ICPP 2018; HiPC 2021): a decoder state is
//                       (bit offset, block within the MCU u, coefficient index k).  Every thread decodes its subsequence from the
//                       state recorded at its start and goes on into the following subsequences, recording its state at each
//                       boundary, until it meets the state already recorded there (at most kWalk subsequences); where several
//                       walks reach one boundary, the one that started furthest upstream wins.  Interval starts are exact; once a
//                       round changes no recorded state, every one is exact (by induction from the interval start), and each round
//                       extends the exact prefix by a whole walk.  After kMaxRounds rounds without a fixed point, dec_serial walks
//                       each unconverged interval with one thread from its exact start, decoding only the subsequences whose
//                       recorded start is still wrong: a stream that never re-synchronises (a table whose codes all have one
//                       length) degrades to serial work that way, but stays exact.
//   5. scan             blocks started per subsequence -> each subsequence's first block in decode order.
//   6. dec_final        the exact decode: i16 AC coefficients into zeroed per-block storage, i32 DC differences, and the first
//                       error / end of data in decode order through one 64-bit atomicMin.
//   7. scan, dec_dc     a per-component prefix sum of the DC differences, restarted at interval starts (the segmented scan is the
//                       plain scan minus its value at the segment start, modulo 2^32 as the i32 predictor wraps), then DC values into
//                       the blocks; blocks after a truncation stay zero.
//   8. dec_recon        one CTA per group of MCUs, 8 threads per block: dequantisation, stb's integer IDCT (:2203-2313), level shift
//                       of component 0, the colour stage of ycbcrToRgbAllBlocks (:2518-2749) and convert_color to the destination.
//
// Semantics follow the reference's bit reader exactly (runs of the 9-bit fast table and the canonical slow path decode the same
// prefix code; running out of bits mid-symbol is the truncation of :2466-2469, which keeps what was decoded).  The one deliberate
// difference is the restart interval: interval i starts at the byte after the i-th RST marker (T.81 F.2.2.5), where the reference
// discards its buffered bits and so decodes every later interval from the wrong bit (DESIGN.md §7).  i32 arithmetic wraps.
#include <cstring>
#include <vector>

#include "zb_convert.cuh"
#include "zb_jpeg_common.cuh"

namespace zb {
namespace {

constexpr int kSubBits = 512;      // bits per subsequence (DESIGN.md §4.9)
constexpr int kMaxRounds = 16;     // synchronisation rounds before the serial walk
constexpr int kWalk = 64;          // subsequences a synchronisation walk may go past its own
constexpr int kChunk = 16;         // bytes per thread of the destuffing pass
constexpr int kMaxBpm = 16;        // blocks per MCU: 4 x 4 for one component
constexpr uint64_t kDead = ~0ull;  // a state past the end of the data

// Decode table of one DHT (parseDHT :1445-1538): fast = len << 8 | symbol for codes of up to 9 bits (0: longer), then F.16's
// maxcode / valptr - mincode per length.
struct __align__(16) DevTable {
    uint16_t fast[512];
    int32_t maxcode[18];
    int32_t valoff[18];
    uint8_t huffval[256];
};
struct Tables { DevTable t[8]; };   // DC 0-3, AC 0-3

struct Zig { uint8_t v[64]; };
constexpr Zig make_zig() {
    Zig z{};
    for (int i = 0; i < 64; ++i) z.v[i] = kZigzag[i];
    return z;
}
__constant__ Zig c_zig = make_zig();

struct Geo {
    uint32_t bw, bh, bwa, bha;      // blocks of the image, and of the MCU-padded image (:1402-1410)
    uint32_t mcu_cols, xs, ys;      // the MCU walk of performBlockScan (:2408-2422)
    uint32_t bpm;                   // blocks per MCU
    uint8_t ucomp[kMaxBpm], uv[kMaxBpm], uh[kMaxBpm], utd[kMaxBpm], uta[kMaxBpm];   // per block of the MCU: component, offset, tables
    uint32_t nc[3], uoff[3];        // blocks per MCU of each component and the first u of each
    uint64_t comp_base[3];          // first DC slot of each component (component-major)
    uint64_t total;                 // blocks in decode order: MCUs x bpm
    uint64_t rblocks;               // blocks per restart interval (0: none)
    uint64_t nblk;                  // bwa x bha
    int ncomp;
};

__device__ __forceinline__ uint32_t bswap(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
// 32 bits of the destuffed stream from bit p (words hold the bytes in memory order; the buffer has two zero words of slack)
__device__ __forceinline__ uint32_t peek32(const uint32_t* __restrict__ w, uint64_t p) {
    const uint64_t i = p >> 5;
    return __funnelshift_l(bswap(w[i + 1]), bswap(w[i]), (uint32_t)(p & 31));
}

// One symbol: code length (0 = no code of up to 16 bits matches) and value.
__device__ __forceinline__ int huff(const DevTable& t, uint32_t w, int* sym) {
    const uint16_t f = t.fast[w >> 23];
    if (f) {
        *sym = f & 0xFF;
        return f >> 8;
    }
    for (int l = 10; l <= 16; ++l) {
        const int32_t code = (int32_t)(w >> (32 - l));
        if (code <= t.maxcode[l]) {
            *sym = t.huffval[(t.valoff[l] + code) & 0xFF];
            return l;
        }
    }
    return 0;
}

// Decoder state (bit offset, block within the MCU, coefficient index; k == 0: the DC is next).
struct St {
    uint64_t p;
    uint32_t uk;   // u << 8 | k
};
__device__ __forceinline__ bool same(St a, St b) { return a.p == b.p && a.uk == b.uk; }

enum { kEvTrunc = 0, kEvError = 1 };

// Decodes from s while the next symbol starts before `end` (FINAL: and, for the last subsequence of an interval, on until the
// interval's blocks are done).  Returns the state reached.  SYNC: *blocks counts the DC symbols started before `end`; errors end
// the block and decoding goes on.  FINAL: coefficients are written and the first event is reported.
template <bool FINAL>
__device__ St decode_run(St s, uint64_t end, uint64_t nbits, const uint32_t* __restrict__ words, const Tables& T, const Geo& g,
                         uint32_t* blocks, uint64_t blk, uint64_t blk_end, bool last, uint64_t sub, int16_t* __restrict__ coef,
                         int32_t* __restrict__ dcdiff, unsigned long long* __restrict__ event) {
    uint64_t p = s.p;
    int u = (int)(s.uk >> 8), k = (int)(s.uk & 0xFF);
    int16_t* cb = nullptr;   // the current block's coefficients (FINAL, in bounds)
    auto locate = [&](uint64_t b) {
        const uint64_t m = b / g.bpm;
        const int uu = (int)(b % g.bpm);
        const uint32_t y = (uint32_t)(m / g.mcu_cols) * g.ys + g.uv[uu], x = (uint32_t)(m % g.mcu_cols) * g.xs + g.uh[uu];
        cb = (y < g.bh && x < g.bw) ? coef + ((uint64_t)g.ucomp[uu] * g.nblk + (uint64_t)y * g.bwa + x) * 64 : nullptr;
    };
    auto report = [&](int kind, bool dc_done) {
        // key: block, then subsequence, then kind (an error and an end of data never share a block and subsequence)
        const unsigned long long key = ((unsigned long long)blk << 32) | ((sub & 0x3FFFFFFFull) << 2) | (dc_done ? 2u : 0u) | kind;
        atomicMin(event, key);
    };
    if (p == kDead || (FINAL && blk >= blk_end)) return s;
    if (FINAL && k > 0) locate(blk);
    for (;;) {
        if (FINAL) {
            if (k == 0 && blk >= blk_end) break;
            if (!last && p >= end) break;
        } else if (p >= end) {
            break;
        }
        const uint64_t avail = p < nbits ? nbits - p : 0;
        if (k == 0) {
            if (FINAL) {
                if (g.utd[u] == 0xFF) { report(kEvError, false); return {kDead, 0}; }
                locate(blk);
            } else {
                ++*blocks;
            }
            const uint32_t w = avail ? peek32(words, p) : 0;
            int sym = 0;
            const int len = g.utd[u] == 0xFF ? 16 : huff(T.t[g.utd[u]], w, &sym);
            if (len == 0 && avail >= 16) {
                if (FINAL) { report(kEvError, false); return {kDead, 0}; }
                p += 16;
                u = (u + 1) % g.bpm;
                continue;
            }
            if (len == 0 || (uint64_t)len > avail) {
                if (FINAL) report(kEvTrunc, false);
                return {kDead, 0};
            }
            if (sym > 11) {
                if (FINAL) { report(kEvError, false); return {kDead, 0}; }
                p += len;
                u = (u + 1) % g.bpm;
                continue;
            }
            if ((uint64_t)(len + sym) > avail) {
                if (FINAL) report(kEvTrunc, false);
                return {kDead, 0};
            }
            if (FINAL) {
                int32_t v = sym ? (int32_t)((w << len) >> (32 - sym)) : 0;
                if (sym && v < (1 << (sym - 1))) v -= (1 << sym) - 1;
                const int c = g.ucomp[u];
                const uint64_t m = blk / g.bpm;
                dcdiff[g.comp_base[c] + m * g.nc[c] + (u - g.uoff[c])] = v;
                if (g.uta[u] == 0xFF) { report(kEvError, true); return {kDead, 0}; }
            }
            p += len + sym;
            k = 1;
            continue;
        }
        const uint32_t w = avail ? peek32(words, p) : 0;
        int sym = 0;
        const int len = g.uta[u] == 0xFF ? 16 : huff(T.t[4 + g.uta[u]], w, &sym);
        bool done = false;
        if (len == 0 && avail >= 16) {
            if (FINAL) { report(kEvError, true); return {kDead, 0}; }
            p += 16;
            done = true;
        } else if (len == 0 || (uint64_t)len > avail) {
            if (FINAL) report(kEvTrunc, true);
            return {kDead, 0};
        } else if (sym == 0) {   // EOB
            p += len;
            done = true;
        } else {
            const int run = sym >> 4, size = sym & 15;
            if (size == 0) {
                if (run != 15) {
                    if (FINAL) { report(kEvError, true); return {kDead, 0}; }
                    p += len;
                    done = true;
                } else {   // ZRL, clipped at 64
                    p += len;
                    k = min(64, k + 16);
                    done = k >= 64;
                }
            } else {
                k += run;
                if (k >= 64) {   // the run ends the block; the magnitude bits are not read (:1300)
                    p += len;
                    done = true;
                } else {
                    if ((uint64_t)(len + size) > avail) {
                        if (FINAL) report(kEvTrunc, true);
                        return {kDead, 0};
                    }
                    if (FINAL && cb) {
                        int32_t v = (int32_t)((w << len) >> (32 - size));
                        if (v < (1 << (size - 1))) v -= (1 << size) - 1;
                        cb[c_zig.v[k]] = (int16_t)v;
                    }
                    p += len + size;
                    ++k;
                    done = k >= 64;
                }
            }
        }
        if (done) {
            u = (u + 1) % (int)g.bpm;
            k = 0;
            if (FINAL) ++blk;
        }
    }
    return {p, (uint32_t)(u << 8 | k)};
}

__device__ __forceinline__ void load_tables(Tables& sh, const Tables* __restrict__ src) {
    const uint4* a = (const uint4*)src;
    uint4* b = (uint4*)&sh;
    for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 16); i += blockDim.x) b[i] = a[i];
    __syncthreads();
}

// ---- stage 1 and 2: scan end, destuffing ------------------------------------------------------------------------------------------

__device__ __forceinline__ bool is_rst(uint8_t b) { return b >= 0xD0 && b <= 0xD7; }

// raw: the bytes after the SOS header (len of them); positions below `limit` (the file's last byte) may end the scan
__global__ void __launch_bounds__(kThreads) dec_scan_end(const uint8_t* __restrict__ raw, uint64_t limit, unsigned long long* __restrict__ end) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= limit) return;
    if (raw[i] == 0xFF) {
        const uint8_t nx = raw[i + 1];
        if (nx != 0x00 && !is_rst(nx)) atomicMin(end, (unsigned long long)i);
    }
}

// Bytes kept and RST markers begun in each chunk of the scan [0, n).  Inside the scan every FF is followed by 00 or an RST.
__global__ void __launch_bounds__(kThreads) dec_destuff_count(const uint8_t* __restrict__ raw, uint64_t n, uint32_t* __restrict__ kept,
                                                               uint32_t* __restrict__ rsts, uint64_t chunks) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= chunks) return;
    uint32_t k = 0, r = 0;
    const uint64_t a = t * kChunk, b = min(n, a + kChunk);
    for (uint64_t i = a; i < b; ++i) {
        const uint8_t v = raw[i];
        const bool second = i > 0 && raw[i - 1] == 0xFF;
        if (v == 0xFF) {
            if (is_rst(raw[i + 1])) ++r;
            else ++k;
        } else if (!second) {
            ++k;
        }
    }
    kept[t] = k;
    rsts[t] = r;
}

__global__ void __launch_bounds__(kThreads) dec_destuff_scatter(const uint8_t* __restrict__ raw, uint64_t n, const uint64_t* __restrict__ koff,
                                                                 const uint64_t* __restrict__ roff, uint64_t chunks, uint8_t* __restrict__ out,
                                                                 uint64_t* __restrict__ rst_at) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= chunks) return;
    uint64_t o = koff[t], r = roff[t];
    const uint64_t a = t * kChunk, b = min(n, a + kChunk);
    for (uint64_t i = a; i < b; ++i) {
        const uint8_t v = raw[i];
        const bool second = i > 0 && raw[i - 1] == 0xFF;
        if (v == 0xFF) {
            if (is_rst(raw[i + 1])) rst_at[r++] = o;
            else out[o++] = 0xFF;
        } else if (!second) {
            out[o++] = v;
        }
    }
}

// ---- stage 3: subsequences -------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint64_t iv_start(uint64_t i, const uint64_t* rst_at) { return i == 0 ? 0 : rst_at[i - 1] * 8; }

__global__ void __launch_bounds__(kThreads) dec_sub_count(uint64_t nint, const uint64_t* __restrict__ rst_at, uint64_t nbits,
                                                          uint32_t* __restrict__ cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nint) return;
    const uint64_t a = iv_start(i, rst_at), b = i + 1 < nint ? iv_start(i + 1, rst_at) : nbits;
    const uint64_t len = b > a ? b - a : 0;
    cnt[i] = (uint32_t)max((uint64_t)1, (len + kSubBits - 1) / kSubBits);
}

// Sub j: the end of its bit range and its interval (found by bisection of the intervals' first subsequences).  The state buffer
// starts at the subsequence starts with u = k = 0, which is exact for interval starts.
__global__ void __launch_bounds__(kThreads) dec_sub_fill(uint64_t nint, uint64_t nsub, const uint64_t* __restrict__ rst_at, uint64_t nbits,
                                                         const uint64_t* __restrict__ first, uint64_t* __restrict__ send,
                                                         uint32_t* __restrict__ siv, St* __restrict__ sa) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nsub) return;
    uint64_t lo = 0, hi = nint;   // the last interval with first[i] <= j
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) / 2;
        if (first[mid] <= j) lo = mid;
        else hi = mid;
    }
    const uint64_t i = lo, a = iv_start(i, rst_at), b = max(a, i + 1 < nint ? iv_start(i + 1, rst_at) : nbits);
    const uint64_t s = a + (j - first[i]) * kSubBits;
    send[j] = j + 1 < first[i + 1] ? s + kSubBits : b;
    siv[j] = (uint32_t)i;
    sa[j] = {s, 0};
}

// ---- stage 4: synchronisation ----------------------------------------------------------------------------------------------------

// One round, in two passes over the same walks (inter-sequence synchronisation).  Thread j decodes subsequence j from a[j], then keeps
// decoding into the following subsequences of its interval as long as the state it reaches at a boundary differs from the one
// recorded there (a), at most kWalk subsequences.  Several walks may reach one boundary; the one that started furthest upstream owns
// it.  PASS 0 claims boundaries (atomicMin of the walker's index); PASS 1 writes each owned boundary's state into b, flags a change,
// and records cnt[j] (blocks started in j from a[j]) and own[j] = the state j itself reaches at j + 1.
// If the exact states end at boundary E, the walker E - 1 starts exact and owns every boundary it reaches (walkers before it stop at
// their first boundary, whose recorded state they confirm), so each round extends the exact prefix by its whole walk.
template <int PASS>
__global__ void __launch_bounds__(kThreads) dec_sync(const Tables* __restrict__ tabs, Geo g, const uint32_t* __restrict__ words, uint64_t nbits,
                                                     uint64_t nsub, const uint64_t* __restrict__ send, const uint32_t* __restrict__ siv,
                                                     const uint64_t* __restrict__ first, const St* __restrict__ a, St* __restrict__ b,
                                                     St* __restrict__ own, uint32_t* __restrict__ owner, uint32_t* __restrict__ cnt,
                                                     int* __restrict__ changed, int* __restrict__ iv_changed) {
    __shared__ Tables T;
    load_tables(T, tabs);
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nsub) return;
    const uint32_t iv = siv[j];
    const uint64_t end = first[iv + 1];
    if (PASS == 1 && j == first[iv]) b[j] = a[j];
    St st = a[j];
    const uint64_t stop = min(end, j + 1 + (uint64_t)kWalk);
    for (uint64_t k = j + 1; k <= stop; ++k) {
        uint32_t n = 0;
        st = decode_run<false>(st, send[k - 1], nbits, words, T, g, &n, 0, 0, false, 0, nullptr, nullptr, nullptr);
        if (PASS == 1 && k == j + 1) {
            cnt[j] = n;
            own[j] = st;
        }
        if (k == end) break;   // past the interval's last subsequence: no boundary to record
        const bool agree = same(st, a[k]);
        if (PASS == 0) {
            atomicMin(owner + k, (uint32_t)j);
        } else if (owner[k] == (uint32_t)j) {
            b[k] = st;
            if (!agree) {
                *changed = 1;
                iv_changed[iv] = 1;
            }
        }
        if (agree) break;
    }
}

// After the last round without a fixed point: cnt[j] counts from old[j] and own[j] is the state reached from old[j] at j + 1.  One
// thread per interval that still changed walks it from its exact start: where its exact state equals old[j], subsequence j's results
// are already exact and are taken; elsewhere it decodes the subsequence itself.  Only streams that never re-synchronise get here.
__global__ void __launch_bounds__(kThreads) dec_serial(const Tables* __restrict__ tabs, Geo g, const uint32_t* __restrict__ words, uint64_t nbits,
                                                       uint64_t nint, const uint64_t* __restrict__ first, const uint64_t* __restrict__ send,
                                                       const St* __restrict__ old, const St* __restrict__ own, St* __restrict__ neu,
                                                       uint32_t* __restrict__ cnt, const int* __restrict__ iv_changed) {
    __shared__ Tables T;
    load_tables(T, tabs);
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nint || !iv_changed[i]) return;
    St s = old[first[i]];
    neu[first[i]] = s;
    for (uint64_t j = first[i]; j < first[i + 1]; ++j) {
        const bool more = j + 1 < first[i + 1];
        if (same(s, old[j])) {
            s = own[j];
        } else {
            uint32_t n = 0;
            s = decode_run<false>(s, send[j], nbits, words, T, g, &n, 0, 0, false, 0, nullptr, nullptr, nullptr);
            cnt[j] = n;
        }
        if (more) neu[j + 1] = s;
    }
}

// ---- stage 6: the exact decode ---------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads) dec_final(const Tables* __restrict__ tabs, Geo g, const uint32_t* __restrict__ words, uint64_t nbits,
                                                      uint64_t nsub, const uint64_t* __restrict__ send, const uint32_t* __restrict__ siv,
                                                      const uint64_t* __restrict__ first, const St* __restrict__ a,
                                                      const uint64_t* __restrict__ boff, int16_t* __restrict__ coef,
                                                      int32_t* __restrict__ dcdiff, unsigned long long* __restrict__ event) {
    __shared__ Tables T;
    load_tables(T, tabs);
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nsub) return;
    const uint64_t iv = siv[j];
    const uint64_t base = g.rblocks ? iv * g.rblocks : 0;
    const uint64_t blk_end = g.rblocks ? min(g.total, base + g.rblocks) : g.total;
    const St s = a[j];
    if (s.p == kDead) return;
    uint64_t blk = base + (boff[j] - boff[first[iv]]);
    if ((s.uk & 0xFF) != 0) --blk;
    const bool last = j + 1 == first[iv + 1];
    decode_run<true>(s, send[j], nbits, words, T, g, nullptr, blk, blk_end, last, j, coef, dcdiff, event);
}

// ---- stage 7: DC values ----------------------------------------------------------------------------------------------------------

// d: a block in decode order.  DC = the prefix sum of its component's differences since the interval start; 0 after a truncation.
__global__ void __launch_bounds__(kThreads) dec_dc(Geo g, const int32_t* __restrict__ dcdiff, const uint64_t* __restrict__ pre,
                                                   uint64_t trunc_blk, int trunc_dc_done, int32_t* __restrict__ dcval, int16_t* __restrict__ coef) {
    const uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= g.total) return;
    const uint64_t m = d / g.bpm;
    const int u = (int)(d % g.bpm), c = g.ucomp[u];
    const uint32_t y = (uint32_t)(m / g.mcu_cols) * g.ys + g.uv[u], x = (uint32_t)(m % g.mcu_cols) * g.xs + g.uh[u];
    if (y >= g.bh || x >= g.bw) return;
    const uint64_t sb = (uint64_t)c * g.nblk + (uint64_t)y * g.bwa + x;
    if (d > trunc_blk || (d == trunc_blk && !trunc_dc_done)) {   // never decoded: the block stays zero
        dcval[sb] = 0;
        if (d > trunc_blk) {
            uint4* q = (uint4*)(coef + sb * 64);
#pragma unroll
            for (int i = 0; i < 8; ++i) q[i] = make_uint4(0, 0, 0, 0);
        }
        return;
    }
    const uint64_t kk = m * g.nc[c] + (u - g.uoff[c]);
    const uint64_t seg = g.rblocks ? (kk / (g.rblocks / g.bpm * g.nc[c])) * (g.rblocks / g.bpm * g.nc[c]) : 0;
    const uint64_t at = g.comp_base[c] + kk, s0 = g.comp_base[c] + seg;
    dcval[sb] = (int32_t)(uint32_t)(pre[at] + (uint32_t)dcdiff[at] - pre[s0]);
}

// ---- stage 8: reconstruction -----------------------------------------------------------------------------------------------------

// idct1D (:2209-2247) in wrapping u32 arithmetic; F2F constants are @round(x * 4096).
__device__ __forceinline__ void idct1d(const int32_t* s, int32_t* o) {
    auto M = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); };
    auto A = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); };
    auto S = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); };
    int32_t p2 = s[2], p3 = s[6];
    int32_t p1 = M(A(p2, p3), 2217);
    int32_t t2 = A(p1, M(p3, -7568));
    int32_t t3 = A(p1, M(p2, 3135));
    p2 = s[0];
    p3 = s[4];
    int32_t t0 = M(A(p2, p3), 4096), t1 = M(S(p2, p3), 4096);
    const int32_t x0 = A(t0, t3), x3 = S(t0, t3), x1 = A(t1, t2), x2 = S(t1, t2);
    t0 = s[7]; t1 = s[5]; t2 = s[3]; t3 = s[1];
    p3 = A(t0, t2);
    int32_t p4 = A(t1, t3);
    p1 = A(t0, t3);
    p2 = A(t1, t2);
    const int32_t p5 = M(A(p3, p4), 4816);
    t0 = M(t0, 1223);
    t1 = M(t1, 8410);
    t2 = M(t2, 12586);
    t3 = M(t3, 6149);
    p1 = A(p5, M(p1, -3686));
    p2 = A(p5, M(p2, -10498));
    p3 = M(p3, -8035);
    p4 = M(p4, -1598);
    t3 = A(t3, A(p1, p4));
    t2 = A(t2, A(p2, p3));
    t1 = A(t1, A(p2, p4));
    t0 = A(t0, A(p1, p3));
    o[0] = x0; o[1] = x1; o[2] = x2; o[3] = x3; o[4] = t0; o[5] = t1; o[6] = t2; o[7] = t3;
}
__device__ __forceinline__ void idct_out(const int32_t* r, int32_t add, int sh, int32_t* w, int stride) {
    auto A = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); };
    auto S = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); };
    const int32_t x0 = A(r[0], add), x1 = A(r[1], add), x2 = A(r[2], add), x3 = A(r[3], add);
    w[0 * stride] = A(x0, r[7]) >> sh; w[1 * stride] = A(x1, r[6]) >> sh;
    w[2 * stride] = A(x2, r[5]) >> sh; w[3 * stride] = A(x3, r[4]) >> sh;
    w[4 * stride] = S(x3, r[4]) >> sh; w[5 * stride] = S(x2, r[5]) >> sh;
    w[6 * stride] = S(x1, r[6]) >> sh; w[7 * stride] = S(x0, r[7]) >> sh;
}

__device__ __forceinline__ uint8_t clamp8(int v) { return (uint8_t)min(max(v, 0), 255); }

// Colour layouts: 0 gray, 1 4:4:4, 2 4:2:2, 3 4:1:1, 4 4:2:0 (the branches of ycbcrToRgbAllBlocks).
template <int LAY> struct Lay {
    static constexpr int H = LAY == 2 ? 2 : (LAY == 3 ? 4 : (LAY == 4 ? 2 : 1)), V = LAY == 4 ? 2 : 1;
    static constexpr int UB = LAY == 0 ? 1 : (LAY == 1 ? 3 : H * V + 2);   // blocks per unit
    static constexpr int UPC = 32 / UB;                                     // units per CTA
};

template <int LAY, int DF>
__global__ void __launch_bounds__(256) dec_recon(Geo g, const int16_t* __restrict__ coef, const int32_t* __restrict__ dcval,
                                                 const uint16_t* __restrict__ qt, uint8_t* __restrict__ dst, uint64_t stride, uint32_t rows,
                                                 uint32_t cols, uint32_t unit_cols, uint32_t unit_rows) {
    using L = Lay<LAY>;
    using CT = typename Fmt<DF>::CT;
    constexpr int PB = (int)sizeof(CT) * Fmt<DF>::N;
    __shared__ int32_t tmp[32][64];
    __shared__ int32_t res[32][64];
    const uint32_t uy = (uint32_t)ZB_GRID_ROW();
    if (uy >= unit_rows) return;
    const uint32_t ux0 = blockIdx.x * L::UPC;

    const int j = threadIdx.x >> 3, r = threadIdx.x & 7;
    const int unit = j / L::UB, b = j % L::UB;
    const uint32_t ux = ux0 + unit;
    int comp = 0;
    uint32_t by = uy * L::V, bx = ux * L::H;
    if (LAY == 1) {
        comp = b;
    } else if (LAY >= 2) {
        if (b < L::H * L::V) {
            by += b / L::H;
            bx += b % L::H;
        } else {
            comp = b - L::H * L::V + 1;
        }
    }
    const bool live = unit < L::UPC && ux < unit_cols && by < g.bha && bx < g.bwa;
    int32_t s[8];
    int32_t nz = 0;
    const uint64_t sb = (uint64_t)comp * g.nblk + (uint64_t)by * g.bwa + bx;
    const uint16_t* q = qt + comp * 64;
#pragma unroll
    for (int v = 0; v < 8; ++v) {
        int32_t c = 0;
        if (live) c = (v == 0 && r == 0) ? dcval[sb] : coef[sb * 64 + v * 8 + r];
        s[v] = (int32_t)((uint32_t)c * q[v * 8 + r]);
        if (v || r) nz |= s[v];
    }
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) nz |= __shfl_xor_sync(0xffffffffu, nz, d);
    const int32_t dc0 = __shfl_sync(0xffffffffu, s[0], threadIdx.x & ~7);
    if (nz) {
        int32_t o[8];
        idct1d(s, o);
        idct_out(o, 512, 10, &tmp[j][r], 8);
    }
    __syncthreads();
    {
        int32_t o[8], w[8];
        if (nz) {
            idct1d(&tmp[j][r * 8], o);
            idct_out(o, 65536, 17, w, 1);
        } else {
            const int32_t v = (int32_t)((uint32_t)dc0 + 4u) >> 3;
#pragma unroll
            for (int x = 0; x < 8; ++x) w[x] = v;
        }
#pragma unroll
        for (int x = 0; x < 8; ++x) res[j][r * 8 + x] = comp == 0 ? (int32_t)((uint32_t)w[x] + 128u) : w[x];
    }
    __syncthreads();

    constexpr int UW = 8 * L::H, UH = 8 * L::V;
    for (int i = threadIdx.x; i < L::UPC * UW * UH; i += blockDim.x) {
        const int un = i / (UW * UH), y = (i / UW) % UH, x = i % UW;
        const uint32_t py = uy * UH + y, px = (ux0 + un) * UW + x;
        if (ux0 + un >= unit_cols || py >= rows || px >= cols) continue;
        const int* blk = res[un * L::UB];
        uint8_t rgb[3];
        CT* o = (CT*)(dst + ((uint64_t)py * stride + px) * PB);
        if constexpr (LAY == 0) {
            const uint8_t gv = clamp8(blk[y * 8 + x]);
            if constexpr (DF == ZB_PIX_U8) o[0] = gv;
            else convert_color<ZB_PIX_U8, DF>(&gv, o);
            continue;
        } else if constexpr (LAY == 1) {
            const int i8 = y * 8 + x;
            const int32_t Y = blk[i8], Cb = res[un * 3 + 1][i8], Cr = res[un * 3 + 2][i8];
            auto M = [](int32_t a, int32_t k) { return (int32_t)((uint32_t)a * (uint32_t)k); };
            auto A = [](int32_t a, int32_t c) { return (int32_t)((uint32_t)a + (uint32_t)c); };
            rgb[0] = clamp8(A(Y, A(M(91881, Cr), 32768) >> 16));
            rgb[1] = clamp8((int32_t)((uint32_t)Y - (uint32_t)(A(A(M(22554, Cb), M(46802, Cr)), 32768) >> 16)));
            rgb[2] = clamp8(A(Y, A(M(116130, Cb), 32768) >> 16));
        } else {
            const int h = x / 8, px8 = x % 8, v = y / 8, py8 = y % 8;
            const int32_t Y = res[un * L::UB + v * L::H + h][py8 * 8 + px8];
            const int32_t* cbb = res[un * L::UB + L::H * L::V];
            const int32_t* crb = res[un * L::UB + L::H * L::V + 1];
            constexpr float sx = L::H == 4 ? 0.25f : 0.5f;
            const float cxf = __fsub_rn(__fmul_rn(__fadd_rn((float)(h * 8 + px8), 0.5f), sx), 0.5f);
            const int cx0 = (int)fminf(fmaxf(floorf(cxf), 0.0f), 7.0f), cx1 = min(7, cx0 + 1);
            const float fx = __fsub_rn(cxf, (float)cx0);
            int32_t Cb, Cr;
            if constexpr (L::V == 1) {
                const float a = (float)cbb[py8 * 8 + cx0], bb = (float)cbb[py8 * 8 + cx1];
                const float c = (float)crb[py8 * 8 + cx0], dd = (float)crb[py8 * 8 + cx1];
                Cb = (int32_t)roundf(__fmaf_rn(__fsub_rn(bb, a), fx, a));
                Cr = (int32_t)roundf(__fmaf_rn(__fsub_rn(dd, c), fx, c));
            } else {
                const float cyf = __fsub_rn(__fmul_rn(__fadd_rn((float)(v * 8 + py8), 0.5f), 0.5f), 0.5f);
                const int cy0 = (int)fminf(fmaxf(floorf(cyf), 0.0f), 7.0f), cy1 = min(7, cy0 + 1);
                const float fy = __fsub_rn(cyf, (float)cy0);
                auto bil = [&](const int32_t* k) {
                    const float k00 = (float)k[cy0 * 8 + cx0], k10 = (float)k[cy0 * 8 + cx1];
                    const float k01 = (float)k[cy1 * 8 + cx0], k11 = (float)k[cy1 * 8 + cx1];
                    const float i0 = __fmaf_rn(__fsub_rn(k10, k00), fx, k00), i1 = __fmaf_rn(__fsub_rn(k11, k01), fx, k01);
                    return (int32_t)roundf(__fmaf_rn(__fsub_rn(i1, i0), fy, i0));
                };
                Cb = bil(cbb);
                Cr = bil(crb);
            }
            // ycbcrToRgb(u8) (color.zig:1057-1068) of the clamped Y, Cb + 128, Cr + 128
            const int64_t Yc = clamp8(Y), B = (int64_t)clamp8(Cb + 128) - 128, R = (int64_t)clamp8(Cr + 128) - 128;
            rgb[0] = clamp8((int)((65536 * Yc + 91881 * R + 32768) >> 16));
            rgb[1] = clamp8((int)((65536 * Yc - 22554 * B - 46802 * R + 32768) >> 16));
            rgb[2] = clamp8((int)((65536 * Yc + 116130 * B + 32768) >> 16));
        }
        if constexpr (LAY != 0) {
            if constexpr (DF == ZB_PIX_RGB8) {
                o[0] = rgb[0]; o[1] = rgb[1]; o[2] = rgb[2];
            } else {
                convert_color<ZB_PIX_RGB8, DF>(rgb, o);
            }
        }
    }
}

// ---- host side --------------------------------------------------------------------------------------------------------------------

struct HTable {
    bool present = false;
    DevTable d;
};
struct Comp { uint8_t id, h, v, tq; };
struct Parsed {
    uint32_t width = 0, height = 0;
    int ncomp = 0;
    bool have_sof = false;
    Comp comps[4] = {};
    HTable tab[8];
    bool have_q[4] = {};
    uint16_t q[4][64] = {};
    int nscan = 0;
    uint8_t scan_id[4], scan_td[4], scan_ta[4];
    uint16_t restart = 0;
    uint32_t bw = 0, bh = 0, bwa = 0, bha = 0;
    uint64_t scan_pos = 0;    // the SOS marker
    uint64_t scan_start = 0;  // first byte after the SOS header
    uint64_t marker_total = 0;
};

zb_jpeg_limits default_limits() { return {100ull << 20, 100ull << 20, 8192, 8192, 67108864ull, 1048576ull, 64}; }
bool exceeds(uint64_t limit, uint64_t v) { return limit != 0 && v > limit; }
uint16_t be16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }

constexpr int kBad = ZB_ERR_INVALID_JPEG, kUns = ZB_ERR_UNSUPPORTED, kBig = ZB_ERR_IMAGE_TOO_LARGE;

int parse_sof(Parsed& st, const uint8_t* d, size_t n, bool progressive, const zb_jpeg_limits& lim) {
    if (st.have_sof) return kBad;   // DuplicateSOF
    if (n < 6) return kBad;
    if (d[0] != 8) return kUns;     // Unsupported12BitPrecision / 16 / UnsupportedPrecision
    st.height = be16(d + 1);
    st.width = be16(d + 3);
    st.ncomp = d[5];
    if (st.width == 0 || st.height == 0) return kBad;
    if (exceeds(lim.max_width, st.width) || exceeds(lim.max_height, st.height)) return kBig;
    if (st.ncomp == 4) return kUns;
    if (st.ncomp != 1 && st.ncomp != 3) return kBad;
    size_t pos = 6;
    int maxh = 0, maxv = 0;
    for (int i = 0; i < st.ncomp; ++i) {
        if (pos + 3 > n) return kBad;
        st.comps[i] = {d[pos], (uint8_t)(d[pos + 1] >> 4), (uint8_t)(d[pos + 1] & 15), d[pos + 2]};
        maxh = maxh > st.comps[i].h ? maxh : st.comps[i].h;
        maxv = maxv > st.comps[i].v ? maxv : st.comps[i].v;
        pos += 3;
    }
    if (maxh > 4 || maxv > 4) return kUns;
    if (st.ncomp == 3) {
        const Comp &y = st.comps[0], &cb = st.comps[1], &cr = st.comps[2];
        if (cb.h != cr.h || cb.v != cr.v) return kBad;
        const bool c11 = cb.h == 1 && cb.v == 1;
        if (!(c11 && ((y.h == 1 && y.v == 1) || (y.h == 2 && y.v == 2) || (y.h == 2 && y.v == 1) || (y.h == 4 && y.v == 1)))) return kUns;
    }
    if (maxh == 0 || maxv == 0) return kBad;
    const uint64_t mw = 8u * maxh, mh = 8u * maxv;
    const uint64_t wa = (st.width + mw - 1) / mw * mw, ha = (st.height + mh - 1) / mh * mh;
    st.bw = (st.width + 7) / 8;
    st.bh = (st.height + 7) / 8;
    st.bwa = (uint32_t)((wa + 7) / 8);
    st.bha = (uint32_t)((ha + 7) / 8);
    if (exceeds(lim.max_pixels, wa * ha)) return kBig;
    if (exceeds(lim.max_blocks, wa * ha / 64)) return kBig;
    st.have_sof = true;
    return progressive ? kUns : ZB_OK;   // progressive frames are this port's limit
}

int parse_dht(Parsed& st, const uint8_t* d, size_t n) {
    if (n == 0) return kBad;
    size_t pos = 0;
    while (pos < n) {
        if (pos + 17 > n) return kBad;
        const int cls = (d[pos] >> 4) & 1, id = d[pos] & 3;
        ++pos;
        const uint8_t* bits = d + pos;
        pos += 16;
        int total = 0;
        for (int i = 0; i < 16; ++i) total += bits[i];
        if (total > 256) return kBad;
        if (pos + total > n) return kBad;
        HTable& t = st.tab[cls * 4 + id];
        std::memset(&t.d, 0, sizeof t.d);
        std::memcpy(t.d.huffval, d + pos, (size_t)total);
        pos += total;
        for (int i = 0; i < 18; ++i) t.d.maxcode[i] = -1;
        uint32_t code = 0;
        int vi = 0;
        for (int i = 0; i < 16; ++i) {
            const int len = i + 1;
            const uint32_t mincode = code;
            const int valptr = vi;
            for (int j = 0; j < bits[i]; ++j) {
                if (code == (1u << len) - 1) return kBad;   // InvalidHuffmanTable
                const uint8_t sym = t.d.huffval[vi++];
                if (len <= 9)
                    for (uint32_t k = 0; k < (1u << (9 - len)); ++k) t.d.fast[(code << (9 - len)) + k] = (uint16_t)(len << 8 | sym);
                ++code;
            }
            if (bits[i]) {
                t.d.maxcode[len] = (int32_t)code - 1;
                t.d.valoff[len] = valptr - (int32_t)mincode;
            }
            code <<= 1;
        }
        t.present = true;
    }
    return ZB_OK;
}

int parse_dqt(Parsed& st, const uint8_t* d, size_t n) {
    if (n == 0) return kBad;
    size_t pos = 0;
    while (pos < n) {
        const int prec = (d[pos] >> 4) & 15, id = d[pos] & 3;
        ++pos;
        const size_t es = prec == 0 ? 1 : 2;
        if (pos + 64 * es > n) return kBad;
        for (int i = 0; i < 64; ++i) st.q[id][kZigzag[i]] = es == 1 ? d[pos + i] : be16(d + pos + 2 * i);
        pos += 64 * es;
        st.have_q[id] = true;
    }
    return ZB_OK;
}

bool known_marker(uint8_t m) { return (m >= 0xC0 && m <= 0xC4) || m == 0xCC || (m >= 0xD0 && m <= 0xEF) || m == 0xFE; }

// decode (:2035-2157) up to the first SOS.  Returns a status; on success st holds the frame, tables and scan.
int parse(Parsed& st, const uint8_t* d, uint64_t len, const zb_jpeg_limits& lim) {
    if (len < 2 || d[0] != 0xFF || d[1] != 0xD8) return kBad;
    if (exceeds(lim.max_jpeg_bytes, len)) return kBig;
    uint64_t pos = 2, total = 0, scans = 0;
    auto payload = [&](const uint8_t** p, size_t* n) {
        if (pos + 4 > len) return kBad;
        const uint16_t l = be16(d + pos + 2);
        if (l < 2 || pos + 2 + l > len) return kBad;
        if (exceeds(lim.max_marker_bytes, total + l)) return kBig;
        total += l;
        *p = d + pos + 4;
        *n = l - 2;
        pos += 2 + (uint64_t)l;
        return (int)ZB_OK;
    };
    int rc;
    while (pos < len - 1) {
        if (d[pos] != 0xFF) return kBad;
        const uint8_t m = d[pos + 1];
        if (!known_marker(m)) {
            pos += 2;
            if (pos + 2 > len) break;
            const uint16_t l = be16(d + pos);
            if (l < 2) return kBad;
            pos += l;
            continue;
        }
        const uint8_t* p;
        size_t n;
        switch (m) {
            case 0xD8: pos += 2; continue;
            case 0xD9: return kBad;   // NoScanData
            case 0xC0: case 0xC2:
                if ((rc = payload(&p, &n)) || (rc = parse_sof(st, p, n, m == 0xC2, lim))) return rc;
                break;
            case 0xC1: case 0xC3: case 0xCC: case 0xDE: case 0xDC: return kUns;
            case 0xC4:
                if ((rc = payload(&p, &n)) || (rc = parse_dht(st, p, n))) return rc;
                break;
            case 0xDB:
                if ((rc = payload(&p, &n)) || (rc = parse_dqt(st, p, n))) return rc;
                break;
            case 0xDD:
                if ((rc = payload(&p, &n))) return rc;
                if (n != 2) return kBad;
                st.restart = be16(p);
                break;
            case 0xDA: {
                if (exceeds(lim.max_scans, scans + 1)) return kBad;   // no scan decoded: NoScanData
                if (pos + 4 > len) return kBad;
                const uint16_t l = be16(d + pos + 2);
                if (l < 2 || pos + 2 + l > len) return kBad;
                const uint8_t* s = d + pos + 4;
                const size_t sn = l - 2;
                if (sn < 6 || s[0] != st.ncomp) return kBad;   // InvalidSOS
                size_t q = 1;
                for (int i = 0; i < st.ncomp; ++i) {
                    if (q + 2 > sn) return kBad;
                    st.scan_id[i] = s[q];
                    st.scan_td[i] = s[q + 1] >> 4;
                    st.scan_ta[i] = s[q + 1] & 15;
                    q += 2;
                }
                if (q + 3 > sn || s[q] != 0 || s[q + 1] != 63 || s[q + 2] != 0) return kBad;
                st.nscan = st.ncomp;
                st.scan_pos = pos;
                st.scan_start = pos + 2 + l;
                st.marker_total = total;
                if (!st.have_sof) return kBad;   // BlockStorageNotAllocated
                return ZB_OK;
            }
            default: {
                if (pos + 4 > len) return kBad;   // NoScanData
                const uint16_t l = be16(d + pos + 2);
                if (exceeds(lim.max_marker_bytes, total + l)) return kBig;
                total += l;
                pos += 2 + (uint64_t)l;
            }
        }
    }
    return kBad;   // NoScanData
}

// MCU walk and per-u tables (performBlockScan :2397-2479).
int geometry(const Parsed& st, Geo& g) {
    std::memset(&g, 0, sizeof g);
    int maxh = 1, maxv = 1;
    for (int i = 0; i < st.ncomp; ++i) {
        maxh = maxh > st.comps[i].h ? maxh : st.comps[i].h;
        maxv = maxv > st.comps[i].v ? maxv : st.comps[i].v;
    }
    const bool nonint = st.nscan == 1 && st.scan_id[0] == 1;
    g.xs = nonint ? 1 : maxh;
    g.ys = nonint ? 1 : maxv;
    g.bw = st.bw; g.bh = st.bh; g.bwa = st.bwa; g.bha = st.bha;
    g.ncomp = st.ncomp;
    g.nblk = (uint64_t)st.bwa * st.bha;
    g.mcu_cols = (st.bw + g.xs - 1) / g.xs;
    const uint64_t mcus = (uint64_t)g.mcu_cols * ((st.bh + g.ys - 1) / g.ys);
    int u = 0;
    for (int c = 0; c < 3; ++c) g.uoff[c] = 0;
    for (int s = 0; s < st.nscan; ++s) {
        int ci = -1;
        for (int i = 0; i < st.ncomp; ++i)
            if (st.comps[i].id == st.scan_id[s]) { ci = i; break; }
        if (ci < 0) return kBad;   // the reference reads undefined sampling factors here
        const int vm = nonint ? 1 : st.comps[ci].v, hm = nonint ? 1 : st.comps[ci].h;
        if (u + vm * hm > kMaxBpm) return kBad;
        if (g.nc[ci] == 0) g.uoff[ci] = u;
        else return kBad;   // a component twice in one scan: its blocks would not be contiguous in the MCU
        g.nc[ci] = vm * hm;
        for (int v = 0; v < vm; ++v)
            for (int h = 0; h < hm; ++h, ++u) {
                g.ucomp[u] = (uint8_t)ci;
                g.uv[u] = (uint8_t)v;
                g.uh[u] = (uint8_t)h;
                g.utd[u] = st.scan_td[s] <= 3 && st.tab[st.scan_td[s]].present ? st.scan_td[s] : 0xFF;
                g.uta[u] = st.scan_ta[s] <= 3 && st.tab[4 + st.scan_ta[s]].present ? st.scan_ta[s] : 0xFF;
            }
    }
    g.bpm = (uint32_t)u;
    uint64_t base = 0;
    for (int c = 0; c < 3; ++c) {
        g.comp_base[c] = base;
        base += mcus * g.nc[c];
    }
    g.total = mcus * g.bpm;
    g.rblocks = (uint64_t)st.restart * g.bpm;
    return ZB_OK;
}

int layout_of(const Parsed& st) {
    if (st.ncomp == 1) return 0;
    const int h = st.comps[0].h, v = st.comps[0].v;
    if (h == 1 && v == 1) return 1;
    if (h == 2 && v == 1) return 2;
    if (h == 4 && v == 1) return 3;
    return 4;
}

template <int LAY, int DF>
int launch_recon_t(const Geo& g, const int16_t* coef, const int32_t* dcval, const uint16_t* qt, zb_image* dst, cudaStream_t s) {
    using L = Lay<LAY>;
    const uint32_t unit_cols = (g.bw + L::H - 1) / L::H, unit_rows = (g.bh + L::V - 1) / L::V;
    const dim3 grid = row_grid(div_up(unit_cols, L::UPC), unit_rows);
    dec_recon<LAY, DF><<<grid, 256, 0, s>>>(g, coef, dcval, qt, (uint8_t*)dst->data, dst->stride, dst->rows, dst->cols, unit_cols, unit_rows);
    ZB_LAUNCHED();
    return ZB_OK;
}
template <int LAY>
int launch_recon_l(int pixfmt, const Geo& g, const int16_t* coef, const int32_t* dcval, const uint16_t* qt, zb_image* dst, cudaStream_t s) {
    switch (pixfmt) {
        case ZB_PIX_U8: return launch_recon_t<LAY, ZB_PIX_U8>(g, coef, dcval, qt, dst, s);
        case ZB_PIX_F32: return launch_recon_t<LAY, ZB_PIX_F32>(g, coef, dcval, qt, dst, s);
        case ZB_PIX_RGB8: return launch_recon_t<LAY, ZB_PIX_RGB8>(g, coef, dcval, qt, dst, s);
        case ZB_PIX_RGBA8: return launch_recon_t<LAY, ZB_PIX_RGBA8>(g, coef, dcval, qt, dst, s);
        default: return launch_recon_t<LAY, ZB_PIX_RGBAF32>(g, coef, dcval, qt, dst, s);
    }
}
int launch_recon(int lay, int pixfmt, const Geo& g, const int16_t* coef, const int32_t* dcval, const uint16_t* qt, zb_image* dst,
                 cudaStream_t s) {
    switch (lay) {
        case 0: return launch_recon_l<0>(pixfmt, g, coef, dcval, qt, dst, s);
        case 1: return launch_recon_l<1>(pixfmt, g, coef, dcval, qt, dst, s);
        case 2: return launch_recon_l<2>(pixfmt, g, coef, dcval, qt, dst, s);
        case 3: return launch_recon_l<3>(pixfmt, g, coef, dcval, qt, dst, s);
        default: return launch_recon_l<4>(pixfmt, g, coef, dcval, qt, dst, s);
    }
}

const char* kernel_name(int lay, int pixfmt) {
    static const char* names[5][5] = {
        {"jpeg_dec_gray_u8", "jpeg_dec_gray_f32", "jpeg_dec_gray_rgb8", "jpeg_dec_gray_rgba8", "jpeg_dec_gray_rgbaf32"},
        {"jpeg_dec_444_u8", "jpeg_dec_444_f32", "jpeg_dec_444_rgb8", "jpeg_dec_444_rgba8", "jpeg_dec_444_rgbaf32"},
        {"jpeg_dec_422_u8", "jpeg_dec_422_f32", "jpeg_dec_422_rgb8", "jpeg_dec_422_rgba8", "jpeg_dec_422_rgbaf32"},
        {"jpeg_dec_411_u8", "jpeg_dec_411_f32", "jpeg_dec_411_rgb8", "jpeg_dec_411_rgba8", "jpeg_dec_411_rgbaf32"},
        {"jpeg_dec_420_u8", "jpeg_dec_420_f32", "jpeg_dec_420_rgb8", "jpeg_dec_420_rgba8", "jpeg_dec_420_rgbaf32"}};
    return names[lay][pixfmt];
}

// bump allocator over one scratch block
struct Carve {
    char* p;
    template <typename T> T* take(uint64_t n) {
        T* r = (T*)p;
        p += (n * sizeof(T) + 255) & ~(uint64_t)255;
        return r;
    }
};

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_jpeg_info(const uint8_t* d, uint64_t len, const zb_jpeg_limits* limits, zb_jpeg_header* out) {
    // getInfo (:77-180) over a fixed reader
    if (!out || (!d && len)) return ZB_ERR_INVALID_ARGUMENT;
    const zb_jpeg_limits lim = limits ? *limits : default_limits();
    uint64_t pos = 0, markers = 0;
#define TAKE(v)                             \
    do {                                    \
        if (pos >= len) return kBad;        \
        (v) = d[pos++];                     \
    } while (0)
    uint8_t a, b;
    TAKE(a);
    TAKE(b);
    if (a != 0xFF || b != 0xD8) return kBad;
    for (;;) {
        for (;;) {
            TAKE(a);
            if (exceeds(lim.max_jpeg_bytes, pos)) return kBig;
            if (a == 0xFF) break;
        }
        TAKE(b);
        while (b == 0xFF) {
            TAKE(b);
            if (exceeds(lim.max_jpeg_bytes, pos)) return kBig;
        }
        if (b == 0x00) continue;
        if (++markers > 10000) return kBig;
        if (b == 0x01 || (b >= 0xD0 && b <= 0xD8)) continue;
        if (b == 0xD9) return kBad;   // MissingSOF
        uint8_t h, l;
        TAKE(h);
        TAKE(l);
        const uint32_t length = (uint32_t)(h << 8 | l);
        if (length < 2) return kBad;
        if (b >= 0xC0 && b <= 0xCF && b != 0xC4 && b != 0xC8 && b != 0xCC) {
            const uint32_t payload = length - 2;
            if (payload < 6) return kBad;
            if (exceeds(lim.max_jpeg_bytes, pos + payload)) return kBig;
            uint8_t p[6];
            for (int i = 0; i < 6; ++i) TAKE(p[i]);
            out->precision = p[0];
            out->height = (uint32_t)(p[1] << 8 | p[2]);
            out->width = (uint32_t)(p[3] << 8 | p[4]);
            out->num_components = p[5];
            out->progressive = b == 0xC2;
            out->subsampling = -1;
            if (p[5] == 3 && payload - 6 >= 9) {
                uint8_t f[9];
                for (int i = 0; i < 9; ++i) TAKE(f[i]);
                if (f[4] == 0x11 && f[7] == 0x11) out->subsampling = f[1] == 0x11 ? 0 : (f[1] == 0x21 ? 1 : (f[1] == 0x22 ? 2 : -1));
            }
            return ZB_OK;
        }
        const uint32_t skip = length - 2;
        if (exceeds(lim.max_jpeg_bytes, pos + skip)) return kBig;
        pos += skip < len - pos ? skip : len - pos;
    }
#undef TAKE
}

extern "C" int zb_jpeg_decode(const uint8_t* data, uint64_t len, const zb_jpeg_limits* limits, zb_image* dst, int pixfmt, zb_stream stream) {
    if (!dst || (!data && len)) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    const zb_jpeg_limits lim = limits ? *limits : default_limits();
    Parsed st;
    int rc = parse(st, data, len, lim);
    if (rc) return rc;
    for (int c = 0; c < st.ncomp; ++c)
        if (st.comps[c].tq > 3 || !st.have_q[st.comps[c].tq]) return kBad;   // MissingQuantTable (dequantizeAllBlocks)
    Geo g;
    if ((rc = geometry(st, g))) return rc;
    if (dst->rows != st.height || dst->cols != st.width) return ZB_ERR_DIMENSION_MISMATCH;
    if (!dst->data || dst->stride < dst->cols) return ZB_ERR_INVALID_ARGUMENT;
    cudaStream_t s = (cudaStream_t)stream;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;

    // the bytes after the SOS header, with slack for the pair test and the 32-bit reads
    const uint64_t L = len - st.scan_start;
    Scratch rawbuf;
    if ((rc = rawbuf.alloc(L + 64, s))) return rc;
    uint8_t* raw = rawbuf.as<uint8_t>();
    ZB_CUDA(cudaMemsetAsync(raw + L, 0, 64, s));
    if (L) ZB_CUDA(cudaMemcpyAsync(raw, data + st.scan_start, L, cudaMemcpyHostToDevice, s));

    // 1. scan end: the first terminating FF below the file's last byte; else the last byte, or the end after a final pair
    uint64_t head[4] = {0, 0, 0, 0};
    Scratch small;
    if ((rc = small.alloc(64, s))) return rc;
    unsigned long long* d_end = small.as<unsigned long long>();
    {
        uint64_t def = 0;
        if (L >= 1) def = L - 1;
        if (L >= 2 && data[len - 2] == 0xFF && (data[len - 1] == 0 || (data[len - 1] >= 0xD0 && data[len - 1] <= 0xD7))) def = L;
        ZB_CUDA(cudaMemcpyAsync(d_end, &def, 8, cudaMemcpyHostToDevice, s));
        if (L >= 2) {
            dec_scan_end<<<div_up(L - 1, kThreads), kThreads, 0, s>>>(raw, L - 1, d_end);
            ZB_LAUNCHED();
        }
    }
    // 2. destuffing
    Scratch ds;
    const uint64_t chunks_max = (L + kChunk - 1) / kChunk + 1, tiles_max = (chunks_max + kScanTile - 1) / kScanTile + 1;
    if ((rc = ds.alloc(chunks_max * 24 + 2 * (chunks_max + 1) * 8 + 2 * tiles_max * 8 + (L + 16) * 8 + (L + 64) + 16 * 256, s))) return rc;
    Carve cv{ds.as<char>()};
    uint32_t* kept = cv.take<uint32_t>(chunks_max);
    uint32_t* rsts = cv.take<uint32_t>(chunks_max);
    uint64_t* koff = cv.take<uint64_t>(chunks_max + 1);
    uint64_t* roff = cv.take<uint64_t>(chunks_max + 1);
    uint64_t* part = cv.take<uint64_t>(tiles_max);
    uint64_t* rst_at = cv.take<uint64_t>(L / 2 + 2);
    uint8_t* stream_b = cv.take<uint8_t>(L + 64);
    ZB_CUDA(cudaMemcpyAsync(&head[0], d_end, 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    const uint64_t E = head[0];
    if (exceeds(lim.max_marker_bytes, st.marker_total + (st.scan_start + E - st.scan_pos))) return kBig;
    const uint64_t chunks = (E + kChunk - 1) / kChunk;
    ZB_CUDA(cudaMemsetAsync(stream_b, 0, L + 64, s));
    uint64_t nb = 0, nrst = 0;
    if (chunks) {
        dec_destuff_count<<<div_up(chunks, kThreads), kThreads, 0, s>>>(raw, E, kept, rsts, chunks);
        ZB_LAUNCHED();
        if ((rc = scan(kept, chunks, part, koff, s)) || (rc = scan(rsts, chunks, part, roff, s))) return rc;
        dec_destuff_scatter<<<div_up(chunks, kThreads), kThreads, 0, s>>>(raw, E, koff, roff, chunks, stream_b, rst_at);
        ZB_LAUNCHED();
        ZB_CUDA(cudaMemcpyAsync(&head[1], koff + chunks, 8, cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaMemcpyAsync(&head[2], roff + chunks, 8, cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        nb = head[1];
        nrst = head[2];
    }
    const uint64_t nbits = nb * 8;
    const uint32_t* words = (const uint32_t*)stream_b;

    // 3. intervals and subsequences
    const uint64_t mcus = g.bpm ? g.total / g.bpm : 0;
    const uint64_t need = st.restart ? (mcus + st.restart - 1) / st.restart : 1;
    const uint64_t nint = need < nrst + 1 ? need : nrst + 1;
    // a missing RST ends the decode at the first block of the interval it would start
    uint64_t event0 = ~0ull;
    if (nint < need) event0 = (nint * g.rblocks) << 32;
    Scratch iv;
    const uint64_t itiles = (nint + kScanTile - 1) / kScanTile + 1;
    if ((rc = iv.alloc(nint * 4 + (nint + 1) * 8 + itiles * 8 + nint * 4 + 16 * 256, s))) return rc;
    Carve ci{iv.as<char>()};
    uint32_t* icnt = ci.take<uint32_t>(nint);
    uint64_t* ifirst = ci.take<uint64_t>(nint + 1);
    uint64_t* ipart = ci.take<uint64_t>(itiles);
    int* iv_changed = ci.take<int>(nint);
    dec_sub_count<<<div_up(nint, kThreads), kThreads, 0, s>>>(nint, rst_at, nbits, icnt);
    ZB_LAUNCHED();
    if ((rc = scan(icnt, nint, ipart, ifirst, s))) return rc;
    ZB_CUDA(cudaMemcpyAsync(&head[3], ifirst + nint, 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    const uint64_t nsub = head[3];

    Scratch sub;
    const uint64_t stiles = (nsub + kScanTile - 1) / kScanTile + 1;
    if ((rc = sub.alloc(nsub * (8 + 8 + 4 + 3 * sizeof(St) + 4 + 4) + (nsub + 1) * 8 + stiles * 8 + sizeof(Tables) + 16 * 256, s))) return rc;
    Carve cs{sub.as<char>()};
    uint64_t* send = cs.take<uint64_t>(nsub);
    uint32_t* siv = cs.take<uint32_t>(nsub);
    St* sa = cs.take<St>(nsub);
    St* sb = cs.take<St>(nsub);
    St* sown = cs.take<St>(nsub);
    uint32_t* owner = cs.take<uint32_t>(nsub);
    uint32_t* cnt = cs.take<uint32_t>(nsub);
    uint64_t* boff = cs.take<uint64_t>(nsub + 1);
    uint64_t* spart = cs.take<uint64_t>(stiles);
    Tables* tabs = cs.take<Tables>(1);
    {
        std::vector<Tables> ht(1);
        std::memset(ht.data(), 0, sizeof(Tables));
        for (int i = 0; i < 8; ++i)
            if (st.tab[i].present) ht[0].t[i] = st.tab[i].d;
        ZB_CUDA(cudaMemcpyAsync(tabs, ht.data(), sizeof(Tables), cudaMemcpyHostToDevice, s));
        ZB_CUDA(cudaStreamSynchronize(s));   // ht is pageable and goes out of scope
    }
    dec_sub_fill<<<div_up(nsub, kThreads), kThreads, 0, s>>>(nint, nsub, rst_at, nbits, ifirst, send, siv, sa);
    ZB_LAUNCHED();

    // 4. synchronisation rounds; flag[0]: some state changed
    int* flag = (int*)(d_end + 1);
    int changed = 1, rounds = 0;
    ZB_CUDA(cudaMemsetAsync(iv_changed, 0, nint * 4, s));
    while (changed && rounds < kMaxRounds) {
        ZB_CUDA(cudaMemsetAsync(flag, 0, 4, s));
        if (rounds + 1 == kMaxRounds) ZB_CUDA(cudaMemsetAsync(iv_changed, 0, nint * 4, s));
        ZB_CUDA(cudaMemsetAsync(owner, 0xFF, nsub * 4, s));
        dec_sync<0><<<div_up(nsub, kThreads), kThreads, 0, s>>>(tabs, g, words, nbits, nsub, send, siv, ifirst, sa, sb, sown, owner, cnt,
                                                                 flag, iv_changed);
        ZB_LAUNCHED();
        dec_sync<1><<<div_up(nsub, kThreads), kThreads, 0, s>>>(tabs, g, words, nbits, nsub, send, siv, ifirst, sa, sb, sown, owner, cnt,
                                                                 flag, iv_changed);
        ZB_LAUNCHED();
        ZB_CUDA(cudaMemcpyAsync(&changed, flag, 4, cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        St* t = sa;
        sa = sb;
        sb = t;
        ++rounds;
    }
    if (changed) {   // no fixed point: walk the intervals that still changed, one thread each
        dec_serial<<<div_up(nint, kThreads), kThreads, 0, s>>>(tabs, g, words, nbits, nint, ifirst, send, sb, sown, sa, cnt, iv_changed);
        ZB_LAUNCHED();
    }

    // 5. first block of each subsequence; 6. the exact decode into zeroed storage
    if ((rc = scan(cnt, nsub, spart, boff, s))) return rc;
    Scratch blk;
    const uint64_t nblk_all = (uint64_t)st.ncomp * g.nblk, dtiles = (g.total + kScanTile - 1) / kScanTile + 1;
    if ((rc = blk.alloc(nblk_all * 128 + nblk_all * 4 + g.total * 4 + (g.total + 1) * 8 + dtiles * 8 + 4 * 64 * 2 + 16 * 256, s))) return rc;
    Carve cb{blk.as<char>()};
    int16_t* coef = cb.take<int16_t>(nblk_all * 64);
    int32_t* dcval = cb.take<int32_t>(nblk_all);
    int32_t* dcdiff = cb.take<int32_t>(g.total);
    uint64_t* pre = cb.take<uint64_t>(g.total + 1);
    uint64_t* dpart = cb.take<uint64_t>(dtiles);
    uint16_t* qt = cb.take<uint16_t>(3 * 64);
    ZB_CUDA(cudaMemsetAsync(coef, 0, nblk_all * 128, s));
    ZB_CUDA(cudaMemsetAsync(dcval, 0, nblk_all * 4, s));   // the MCU-padding blocks are never decoded but are read by dec_recon
    ZB_CUDA(cudaMemsetAsync(dcdiff, 0, g.total * 4, s));
    unsigned long long* d_event = (unsigned long long*)(d_end + 2);
    ZB_CUDA(cudaMemcpyAsync(d_event, &event0, 8, cudaMemcpyHostToDevice, s));
    dec_final<<<div_up(nsub, kThreads), kThreads, 0, s>>>(tabs, g, words, nbits, nsub, send, siv, ifirst, sa, boff, coef, dcdiff, d_event);
    ZB_LAUNCHED();
    uint64_t event = 0;
    ZB_CUDA(cudaMemcpyAsync(&event, d_event, 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    if (event != ~0ull && (event & 1)) return kBad;
    const uint64_t trunc_blk = event == ~0ull ? ~0ull : event >> 32;
    const int trunc_dc = event == ~0ull ? 1 : (int)((event >> 1) & 1);

    // 7. DC values
    if ((rc = scan((const uint32_t*)dcdiff, g.total, dpart, pre, s))) return rc;
    dec_dc<<<div_up(g.total, kThreads), kThreads, 0, s>>>(g, dcdiff, pre, trunc_blk, trunc_dc, dcval, coef);
    ZB_LAUNCHED();

    // 8. reconstruction
    {
        uint16_t hq[3][64] = {};
        for (int c = 0; c < st.ncomp; ++c) std::memcpy(hq[c], st.q[st.comps[c].tq], 128);
        ZB_CUDA(cudaMemcpyAsync(qt, hq, sizeof hq, cudaMemcpyHostToDevice, s));
        const int lay = layout_of(st);
        if ((rc = launch_recon(lay, pixfmt, g, coef, dcval, qt, dst, s))) return rc;
        t_last_kernel = kernel_name(lay, pixfmt);
        ZB_CUDA(cudaStreamSynchronize(s));   // hq is on this frame
    }
    return ZB_OK;
}
