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
// zb_jpeg_decode_batch runs these stages once for many files (zb_jpeg_decode is its batch of one): the scans are packed into one
// buffer, intervals and subsequences are numbered over the batch, each CTA of the per-subsequence kernels serves one file, and each
// file keeps its own event slot (DESIGN.md §4.9, "Batches").
//
// Semantics follow the reference's bit reader exactly (runs of the 9-bit fast table and the canonical slow path decode the same
// prefix code; running out of bits mid-symbol is the truncation of :2466-2469, which keeps what was decoded).  The one deliberate
// difference is the restart interval: interval i starts at the byte after the i-th RST marker (T.81 F.2.2.5), where the reference
// discards its buffered bits and so decodes every later interval from the wrong bit (DESIGN.md §7).  i32 arithmetic wraps.
#include <algorithm>
#include <cstring>
#include <memory>
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

struct __align__(16) Geo {
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
    // where the file lies in its batch
    uint64_t bit0, bitend;          // its destuffed stream in the batch's bit stream
    uint64_t rst0, nint, ibase;     // its first RST slot, its restart intervals and the batch index of the first
    uint64_t coef0, dc0;            // its first block slot (coef, dcval) and its first DC difference slot
    uint8_t* dst;                   // the destination image
    uint64_t dstride;
    uint32_t rows, cols;
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
// interval's blocks are done).  The file's stream ends at g.bitend.  Returns the state reached.  SYNC: *blocks counts the DC symbols started before `end`; errors end
// the block and decoding goes on.  FINAL: coefficients are written and the first event is reported.
template <bool FINAL>
__device__ St decode_run(St s, uint64_t end, const uint32_t* __restrict__ words, const Tables& T, const Geo& g,
                         uint32_t* blocks, uint64_t blk, uint64_t blk_end, bool last, uint64_t sub, int16_t* __restrict__ coef,
                         int32_t* __restrict__ dcdiff, unsigned long long* __restrict__ event) {
    // the walks are latency-bound: the scalars read on every symbol stay in registers, not in the shared Geo
    const uint64_t nbits = g.bitend;
    const int bpm = (int)g.bpm;
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
                u = (u + 1) % bpm;
                continue;
            }
            if (len == 0 || (uint64_t)len > avail) {
                if (FINAL) report(kEvTrunc, false);
                return {kDead, 0};
            }
            if (sym > 11) {
                if (FINAL) { report(kEvError, false); return {kDead, 0}; }
                p += len;
                u = (u + 1) % bpm;
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
            u = (u + 1) % bpm;
            k = 0;
            if (FINAL) ++blk;
        }
    }
    return {p, (uint32_t)(u << 8 | k)};
}

// The per-subsequence and per-interval kernels give each CTA the items of one file (a host-built table of Cta); the CTA stages
// that file's tables and geometry in shared memory.
struct Cta {
    uint64_t first, end;   // items [first, end)
    uint64_t file;
};
__device__ __forceinline__ void load_file(Tables& shT, Geo& shG, const Tables* __restrict__ tabs, const Geo* __restrict__ geos, uint64_t f0) {
    const uint4* a = (const uint4*)(tabs + f0);
    uint4* b = (uint4*)&shT;
    for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 16); i += blockDim.x) b[i] = a[i];
    const uint4* c = (const uint4*)(geos + f0);
    uint4* d = (uint4*)&shG;
    for (int i = threadIdx.x; i < (int)(sizeof(Geo) / 16); i += blockDim.x) d[i] = c[i];
    __syncthreads();
}

// The last i < n with first[i] <= x (first ascending, first[0] <= x): the file, interval or segment that item x belongs to.
__device__ __forceinline__ uint64_t last_le(const uint64_t* __restrict__ first, uint64_t n, uint64_t x) {
    uint64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) / 2;
        if (first[mid] <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}

// ---- stage 1 and 2: scan end, destuffing ------------------------------------------------------------------------------------------

__device__ __forceinline__ bool is_rst(uint8_t b) { return b >= 0xD0 && b <= 0xD7; }

// raw: the packed bytes after each file's SOS header (nf files, file f at foff[f], foff[nf] = total); positions of file f below
// flim[f] (its last byte) may end its scan.  Each file is followed by zeros, so raw[i + 1] never reads the next file.
__global__ void __launch_bounds__(kThreads) dec_scan_end(const uint8_t* __restrict__ raw, const uint64_t* __restrict__ foff,
                                                         const uint64_t* __restrict__ flim, uint64_t nf, unsigned long long* __restrict__ end) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= foff[nf] || raw[i] != 0xFF) return;
    const uint64_t f = last_le(foff, nf, i), at = i - foff[f];
    if (at >= flim[f]) return;
    const uint8_t nx = raw[i + 1];
    if (nx != 0x00 && !is_rst(nx)) atomicMin(end + f, (unsigned long long)at);
}

// The scans of nf files, cut into chunks of kChunk bytes numbered over the batch: file f's scan is raw[off[f], off[f] + len[f]) and
// its chunks start at cfirst[f].
struct Chunks {
    const uint64_t* cfirst;   // nf + 1
    const uint64_t* off;
    const uint64_t* len;
    uint64_t nf;
};

// Bytes kept and RST markers begun in each chunk.  Inside the scan every FF is followed by 00 or an RST.
__global__ void __launch_bounds__(kThreads) dec_destuff_count(const uint8_t* __restrict__ raw, Chunks c, uint32_t* __restrict__ kept,
                                                               uint32_t* __restrict__ rsts) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= c.cfirst[c.nf]) return;
    const uint64_t f = last_le(c.cfirst, c.nf, t), n = c.len[f];
    const uint8_t* r = raw + c.off[f];
    uint32_t k = 0, q = 0;
    const uint64_t a = (t - c.cfirst[f]) * kChunk, b = min(n, a + kChunk);
    for (uint64_t i = a; i < b; ++i) {
        const uint8_t v = r[i];
        const bool second = i > 0 && r[i - 1] == 0xFF;
        if (v == 0xFF) {
            if (is_rst(r[i + 1])) ++q;
            else ++k;
        } else if (!second) {
            ++k;
        }
    }
    kept[t] = k;
    rsts[t] = q;
}

// File f's destuffed stream goes to out + off[f] (the same offset as its raw bytes: it is no longer); each RST's destuffed offset
// within its file goes to rst_at at the marker's batch index.
__global__ void __launch_bounds__(kThreads) dec_destuff_scatter(const uint8_t* __restrict__ raw, Chunks c, const uint64_t* __restrict__ koff,
                                                                 const uint64_t* __restrict__ roff, uint8_t* __restrict__ out,
                                                                 uint64_t* __restrict__ rst_at) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= c.cfirst[c.nf]) return;
    const uint64_t f = last_le(c.cfirst, c.nf, t), n = c.len[f];
    const uint8_t* r = raw + c.off[f];
    uint8_t* w = out + c.off[f];
    uint64_t o = koff[t] - koff[c.cfirst[f]], q = roff[t];
    const uint64_t a = (t - c.cfirst[f]) * kChunk, b = min(n, a + kChunk);
    for (uint64_t i = a; i < b; ++i) {
        const uint8_t v = r[i];
        const bool second = i > 0 && r[i - 1] == 0xFF;
        if (v == 0xFF) {
            if (is_rst(r[i + 1])) rst_at[q++] = o;
            else w[o++] = 0xFF;
        } else if (!second) {
            w[o++] = v;
        }
    }
}

// out[i] = src[at[i]], i < n: a scan's value at each file's first item (and its total), for the host.
__global__ void dec_pick(const uint64_t* __restrict__ at, uint64_t n, const uint64_t* __restrict__ src, uint64_t* __restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = src[at[i]];
}

// ---- stage 3: intervals and subsequences -----------------------------------------------------------------------------------------

// Interval i of the batch (file f's intervals start at ibase[f]): its bit range [ia, ib) and its subsequence count.
__global__ void __launch_bounds__(kThreads) dec_iv_fill(const Geo* __restrict__ geos, const uint64_t* __restrict__ ibase, uint64_t nf,
                                                        const uint64_t* __restrict__ rst_at, uint64_t* __restrict__ ia, uint64_t* __restrict__ ib,
                                                        uint32_t* __restrict__ cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ibase[nf]) return;
    const uint64_t f = last_le(ibase, nf, i), li = i - ibase[f];
    const Geo& g = geos[f];
    const uint64_t a = g.bit0 + (li ? rst_at[g.rst0 + li - 1] * 8 : 0);
    const uint64_t b = max(a, li + 1 < g.nint ? g.bit0 + rst_at[g.rst0 + li] * 8 : g.bitend);
    ia[i] = a;
    ib[i] = b;
    cnt[i] = (uint32_t)max((uint64_t)1, (b - a + kSubBits - 1) / kSubBits);
}

// Sub j: the end of its bit range and its interval (found by bisection of the intervals' first subsequences).  The state buffer
// starts at the subsequence starts with u = k = 0, which is exact for interval starts.
__global__ void __launch_bounds__(kThreads) dec_sub_fill(uint64_t nint, uint64_t nsub, const uint64_t* __restrict__ ia,
                                                         const uint64_t* __restrict__ ib, const uint64_t* __restrict__ first,
                                                         uint64_t* __restrict__ send, uint32_t* __restrict__ siv, St* __restrict__ sa) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nsub) return;
    const uint64_t i = last_le(first, nint, j);
    const uint64_t s = ia[i] + (j - first[i]) * kSubBits;
    send[j] = j + 1 < first[i + 1] ? s + kSubBits : ib[i];
    siv[j] = (uint32_t)i;
    sa[j] = {s, 0};
}

// ---- stage 4: synchronisation ----------------------------------------------------------------------------------------------------

// What the per-subsequence kernels read of the batch.
struct Pool {
    const Tables* tabs;
    const Geo* geos;
    const Cta* ctas;          // CTA -> one file's subsequences (dec_sync, dec_final) or intervals (dec_serial)
    const uint32_t* words;    // the destuffed streams
    const uint64_t* send;     // subsequence -> end bit
    const uint32_t* siv;      // subsequence -> interval
    const uint64_t* first;    // interval -> first subsequence (nint + 1)
};

// One round, in two passes over the same walks (inter-sequence synchronisation).  Thread j decodes subsequence j from a[j], then keeps
// decoding into the following subsequences of its interval as long as the state it reaches at a boundary differs from the one
// recorded there (a), at most kWalk subsequences.  Several walks may reach one boundary; the one that started furthest upstream owns
// it.  PASS 0 claims boundaries (atomicMin of the walker's index); PASS 1 writes each owned boundary's state into b, flags a change,
// and records cnt[j] (blocks started in j from a[j]) and own[j] = the state j itself reaches at j + 1.
// If the exact states end at boundary E, the walker E - 1 starts exact and owns every boundary it reaches (walkers before it stop at
// their first boundary, whose recorded state they confirm), so each round extends the exact prefix by its whole walk.  No walk
// leaves its interval, so the intervals of every file of the batch run in one pool.
template <int PASS>
__global__ void __launch_bounds__(kThreads) dec_sync(Pool P, const St* __restrict__ a, St* __restrict__ b, St* __restrict__ own,
                                                     uint32_t* __restrict__ owner, uint32_t* __restrict__ cnt, int* __restrict__ changed,
                                                     int* __restrict__ iv_changed) {
    __shared__ Tables T;
    __shared__ Geo g;
    const Cta c = P.ctas[blockIdx.x];
    load_file(T, g, P.tabs, P.geos, c.file);
    const uint64_t j = c.first + threadIdx.x;
    if (j >= c.end) return;
    const uint32_t iv = P.siv[j];
    const uint64_t end = P.first[iv + 1];
    if (PASS == 1 && j == P.first[iv]) b[j] = a[j];
    St st = a[j];
    const uint64_t stop = min(end, j + 1 + (uint64_t)kWalk);
    for (uint64_t k = j + 1; k <= stop; ++k) {
        uint32_t n = 0;
        st = decode_run<false>(st, P.send[k - 1], P.words, T, g, &n, 0, 0, false, 0, nullptr, nullptr, nullptr);
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
__global__ void __launch_bounds__(kThreads) dec_serial(Pool P, const St* __restrict__ old, const St* __restrict__ own, St* __restrict__ neu,
                                                       uint32_t* __restrict__ cnt, const int* __restrict__ iv_changed) {
    __shared__ Tables T;
    __shared__ Geo g;
    const Cta c = P.ctas[blockIdx.x];
    load_file(T, g, P.tabs, P.geos, c.file);
    const uint64_t i = c.first + threadIdx.x;
    if (i >= c.end || !iv_changed[i]) return;
    const uint64_t j0 = P.first[i], j1 = P.first[i + 1];
    St s = old[j0];
    neu[j0] = s;
    for (uint64_t j = j0; j < j1; ++j) {
        const bool more = j + 1 < j1;
        if (same(s, old[j])) {
            s = own[j];
        } else {
            uint32_t n = 0;
            s = decode_run<false>(s, P.send[j], P.words, T, g, &n, 0, 0, false, 0, nullptr, nullptr, nullptr);
            cnt[j] = n;
        }
        if (more) neu[j + 1] = s;
    }
}

// ---- stage 6: the exact decode ---------------------------------------------------------------------------------------------------

// event[f]: file f's first error or end of data.
__global__ void __launch_bounds__(kThreads) dec_final(Pool P, const St* __restrict__ a, const uint64_t* __restrict__ boff,
                                                      int16_t* __restrict__ coef, int32_t* __restrict__ dcdiff,
                                                      unsigned long long* __restrict__ event) {
    __shared__ Tables T;
    __shared__ Geo g;
    const Cta c = P.ctas[blockIdx.x];
    load_file(T, g, P.tabs, P.geos, c.file);
    const uint64_t j = c.first + threadIdx.x;
    if (j >= c.end) return;
    const uint64_t iv = P.siv[j];
    const uint64_t base = g.rblocks ? (iv - g.ibase) * g.rblocks : 0;
    const uint64_t blk_end = g.rblocks ? min(g.total, base + g.rblocks) : g.total;
    const St s = a[j];
    if (s.p == kDead) return;
    uint64_t blk = base + (boff[j] - boff[P.first[iv]]);
    if ((s.uk & 0xFF) != 0) --blk;
    const bool last = j + 1 == P.first[iv + 1];
    decode_run<true>(s, P.send[j], P.words, T, g, nullptr, blk, blk_end, last, j, coef + g.coef0 * 64, dcdiff + g.dc0, event + c.file);
}

// ---- stage 7: DC values ----------------------------------------------------------------------------------------------------------

__host__ __device__ __forceinline__ bool failed(unsigned long long e) { return e != ~0ull && (e & 1); }

// d: a block in decode order over the batch (file f's blocks start at dfirst[f]).  DC = the prefix sum of its component's
// differences since the interval start; 0 after a truncation.  Files whose decode failed are skipped.
__global__ void __launch_bounds__(kThreads) dec_dc(const Geo* __restrict__ geos, const uint64_t* __restrict__ dfirst, uint64_t nf,
                                                   const int32_t* __restrict__ dcdiff, const uint64_t* __restrict__ pre,
                                                   const unsigned long long* __restrict__ event, int32_t* __restrict__ dcval,
                                                   int16_t* __restrict__ coef) {
    const uint64_t dd = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (dd >= dfirst[nf]) return;
    const uint64_t f = last_le(dfirst, nf, dd), d = dd - dfirst[f];
    const unsigned long long e = event[f];
    if (failed(e)) return;
    const uint64_t trunc_blk = e == ~0ull ? ~0ull : e >> 32;
    const bool trunc_dc_done = e == ~0ull || ((e >> 1) & 1);
    const Geo& g = geos[f];
    const uint64_t m = d / g.bpm;
    const int u = (int)(d % g.bpm), c = g.ucomp[u];
    const uint32_t y = (uint32_t)(m / g.mcu_cols) * g.ys + g.uv[u], x = (uint32_t)(m % g.mcu_cols) * g.xs + g.uh[u];
    if (y >= g.bh || x >= g.bw) return;
    const uint64_t sb = g.coef0 + (uint64_t)c * g.nblk + (uint64_t)y * g.bwa + x;
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
    const uint64_t at = g.dc0 + g.comp_base[c] + kk, s0 = g.dc0 + g.comp_base[c] + seg;
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

// One CTA per (row tile, group of units): tiles[t] = (file, unit row), for every file of the batch with this layout and pixel format.
// Files whose decode failed are left untouched.
template <int LAY, int DF>
__global__ void __launch_bounds__(256) dec_recon(const Geo* __restrict__ geos, const uint2* __restrict__ tiles, uint32_t ntiles,
                                                 const int16_t* __restrict__ coef_all, const int32_t* __restrict__ dcval_all,
                                                 const uint16_t* __restrict__ qt_all, const unsigned long long* __restrict__ event) {
    using L = Lay<LAY>;
    using CT = typename Fmt<DF>::CT;
    constexpr int PB = (int)sizeof(CT) * Fmt<DF>::N;
    __shared__ int32_t tmp[32][64];
    __shared__ int32_t res[32][64];
    const uint32_t t = (uint32_t)ZB_GRID_ROW();
    if (t >= ntiles) return;
    const uint2 tile = tiles[t];
    const Geo& g = geos[tile.x];
    const uint32_t uy = tile.y, unit_cols = (g.bw + L::H - 1) / L::H;
    const uint32_t ux0 = blockIdx.x * L::UPC;
    if (ux0 >= unit_cols || failed(event[tile.x])) return;
    const int16_t* __restrict__ coef = coef_all + g.coef0 * 64;
    const int32_t* __restrict__ dcval = dcval_all + g.coef0;
    const uint16_t* __restrict__ qt = qt_all + (uint64_t)tile.x * 3 * 64;
    uint8_t* __restrict__ dst = g.dst;
    const uint64_t stride = g.dstride;
    const uint32_t rows = g.rows, cols = g.cols;

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

// Units (MCU columns of the colour stage) per layout, as Lay<> has them.
constexpr int kLayH[5] = {1, 1, 2, 4, 2}, kLayV[5] = {1, 1, 1, 1, 2};
static_assert(kLayH[2] == Lay<2>::H && kLayH[3] == Lay<3>::H && kLayH[4] == Lay<4>::H && kLayV[4] == Lay<4>::V, "layout units");

struct Recon {
    const Geo* geos;
    const uint2* tiles;
    uint32_t ntiles, max_unit_cols;
    const int16_t* coef;
    const int32_t* dcval;
    const uint16_t* qt;
    const unsigned long long* event;
};

template <int LAY>
int launch_recon_l(int pixfmt, const Recon& r, cudaStream_t s) {
    const dim3 grid = row_grid(div_up(r.max_unit_cols, Lay<LAY>::UPC), r.ntiles);
    return dispatch_pixfmt<kFmtAll>(pixfmt, [&](auto f) -> int {
        dec_recon<LAY, decltype(f)::value><<<grid, 256, 0, s>>>(r.geos, r.tiles, r.ntiles, r.coef, r.dcval, r.qt, r.event);
        ZB_LAUNCHED();
        return ZB_OK;
    });
}
int launch_recon(int lay, int pixfmt, const Recon& r, cudaStream_t s) {
    switch (lay) {
        case 0: return launch_recon_l<0>(pixfmt, r, s);
        case 1: return launch_recon_l<1>(pixfmt, r, s);
        case 2: return launch_recon_l<2>(pixfmt, r, s);
        case 3: return launch_recon_l<3>(pixfmt, r, s);
        default: return launch_recon_l<4>(pixfmt, r, s);
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

// Every stage runs once for the whole batch: the files' scans are packed into one buffer, their restart intervals form one pool of
// subsequences, and the host waits for the scan ends, the destuffed lengths, the subsequence count, each synchronisation round and
// the end, whatever the number of files (DESIGN.md §4.9).
extern "C" int zb_jpeg_decode_batch(uint32_t n, const uint8_t* const* data, const uint64_t* len, const zb_jpeg_limits* limits,
                                    zb_image* dst, const int* pixfmt, int* status, zb_stream stream) {
    if (n == 0) return ZB_OK;
    if (!data || !len || !dst || !pixfmt || !status) return ZB_ERR_INVALID_ARGUMENT;
    const zb_jpeg_limits lim = limits ? *limits : default_limits();
    cudaStream_t s = (cudaStream_t)stream;
    int rc;

    // host: each file's segments before its SOS.  A file refused here is never touched.
    struct Job {
        uint32_t i;              // index in the call
        int lay;
        uint16_t restart;
        uint64_t scan_pos, marker_total, scan_start, L;   // L: the bytes after the SOS header
        uint64_t off;            // where they start in the packed buffer (a multiple of 16)
    };
    std::vector<Job> jobs;
    std::vector<Geo> geos;
    std::vector<Tables> tabs;
    std::vector<uint16_t> qts;   // 3 x 64 per job: the component's quantisation table, natural order
    jobs.reserve(n);
    geos.reserve(n);
    tabs.reserve(n);
    auto prepare = [&](uint32_t i) -> int {
        if (!data[i] && len[i]) return ZB_ERR_INVALID_ARGUMENT;
        if (!pixfmt_in(kFmtAll, pixfmt[i])) return ZB_ERR_UNSUPPORTED;
        Parsed st;
        int r = parse(st, data[i], len[i], lim);
        if (r) return r;
        for (int c = 0; c < st.ncomp; ++c)
            if (st.comps[c].tq > 3 || !st.have_q[st.comps[c].tq]) return kBad;   // MissingQuantTable (dequantizeAllBlocks)
        Geo g;
        if ((r = geometry(st, g))) return r;
        const zb_image& d = dst[i];
        if (d.rows != st.height || d.cols != st.width) return ZB_ERR_DIMENSION_MISMATCH;
        if (!d.data || d.stride < d.cols) return ZB_ERR_INVALID_ARGUMENT;
        g.dst = (uint8_t*)d.data;
        g.dstride = d.stride;
        g.rows = d.rows;
        g.cols = d.cols;
        geos.push_back(g);
        jobs.push_back({i, layout_of(st), st.restart, st.scan_pos, st.marker_total, st.scan_start, len[i] - st.scan_start, 0});
        tabs.emplace_back();
        std::memset(&tabs.back(), 0, sizeof(Tables));
        for (int k = 0; k < 8; ++k)
            if (st.tab[k].present) tabs.back().t[k] = st.tab[k].d;
        qts.resize(qts.size() + 3 * 64, 0);
        for (int c = 0; c < st.ncomp; ++c) std::memcpy(&qts[qts.size() - 3 * 64 + c * 64], st.q[st.comps[c].tq], 128);
        return ZB_OK;
    };
    for (uint32_t i = 0; i < n; ++i) status[i] = prepare(i);
    if (jobs.empty()) return ZB_OK;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;

    // 0. one upload: each file's bytes after its SOS header at a multiple of 16, followed by at least 64 zero bytes (the pair test
    //    and the 32-bit reads of the last word never reach the next file)
    const uint64_t na = jobs.size();
    std::vector<uint64_t> ha(3 * na + 1);   // packed offsets (na + 1), the positions that may end each scan, scan-end defaults
    uint64_t total = 0;
    for (uint64_t a = 0; a < na; ++a) {
        Job& jb = jobs[a];
        jb.off = ha[a] = total;
        total += (jb.L + 64 + 15) & ~(uint64_t)15;
        ha[na + 1 + a] = jb.L >= 2 ? jb.L - 1 : 0;
        // the first terminating FF below the file's last byte; else the last byte, or the end after a final pair
        const uint8_t* d = data[jb.i];
        const uint64_t ln = len[jb.i];
        uint64_t def = jb.L >= 1 ? jb.L - 1 : 0;
        if (jb.L >= 2 && d[ln - 2] == 0xFF && (d[ln - 1] == 0 || (d[ln - 1] >= 0xD0 && d[ln - 1] <= 0xD7))) def = jb.L;
        ha[2 * na + 1 + a] = def;
    }
    ha[na] = total;
    Scratch rawbuf, meta_a;
    if ((rc = rawbuf.alloc(total, s)) || (rc = meta_a.alloc(ha.size() * 8, s))) return rc;
    uint8_t* raw = rawbuf.as<uint8_t>();
    uint64_t* d_ha = meta_a.as<uint64_t>();
    std::unique_ptr<uint8_t[]> pack;
    if (na == 1) {   // the packed buffer is the file itself
        const Job& jb = jobs[0];
        ZB_CUDA(cudaMemsetAsync(raw + jb.L, 0, total - jb.L, s));
        if (jb.L) ZB_CUDA(cudaMemcpyAsync(raw, data[jb.i] + jb.scan_start, jb.L, cudaMemcpyHostToDevice, s));
    } else {
        pack.reset(new uint8_t[total]);
        for (uint64_t a = 0; a < na; ++a) {
            const Job& jb = jobs[a];
            if (jb.L) std::memcpy(pack.get() + jb.off, data[jb.i] + jb.scan_start, jb.L);
            std::memset(pack.get() + jb.off + jb.L, 0, ha[a + 1] - jb.off - jb.L);
        }
        ZB_CUDA(cudaMemcpyAsync(raw, pack.get(), total, cudaMemcpyHostToDevice, s));
    }
    ZB_CUDA(cudaMemcpyAsync(d_ha, ha.data(), ha.size() * 8, cudaMemcpyHostToDevice, s));

    // 1. scan ends, and MarkerDataLimitExceeded per file
    unsigned long long* d_end = (unsigned long long*)(d_ha + 2 * na + 1);
    dec_scan_end<<<div_up(total, kThreads), kThreads, 0, s>>>(raw, d_ha, d_ha + na + 1, na, d_end);
    ZB_LAUNCHED();
    std::vector<uint64_t> E(na);
    ZB_CUDA(cudaMemcpyAsync(E.data(), d_end, na * 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> plan;   // the jobs that go on
    for (uint32_t a = 0; a < na; ++a) {
        const Job& jb = jobs[a];
        if (exceeds(lim.max_marker_bytes, jb.marker_total + (jb.scan_start + E[a] - jb.scan_pos))) status[jb.i] = kBig;
        else plan.push_back(a);
    }
    if (plan.empty()) return ZB_OK;
    const uint64_t nf = plan.size();

    // 2. destuffing: file f's stream lands at its packed offset, so it starts on a word and keeps the zeros that follow it
    std::vector<uint64_t> hb(3 * nf + 1);   // first chunk of each file (nf + 1), packed offsets, scan lengths
    for (uint64_t f = 0; f < nf; ++f) {
        hb[f + 1] = hb[f] + (E[plan[f]] + kChunk - 1) / kChunk;
        hb[nf + 1 + f] = jobs[plan[f]].off;
        hb[2 * nf + 1 + f] = E[plan[f]];
    }
    const uint64_t chunks = hb[nf], tiles = (chunks + kScanTile - 1) / kScanTile + 1;
    Scratch ds;
    if ((rc = ds.alloc(chunks * 8 + 2 * (chunks + 1) * 8 + tiles * 8 + (total / 2 + 2) * 8 + total + hb.size() * 8 + 2 * (nf + 1) * 8 + 8 * 256,
                       s)))
        return rc;
    Carve cv{ds.as<char>()};
    uint32_t* kept = cv.take<uint32_t>(chunks);
    uint32_t* rsts = cv.take<uint32_t>(chunks);
    uint64_t* koff = cv.take<uint64_t>(chunks + 1);
    uint64_t* roff = cv.take<uint64_t>(chunks + 1);
    uint64_t* part = cv.take<uint64_t>(tiles);
    uint64_t* rst_at = cv.take<uint64_t>(total / 2 + 2);
    uint8_t* stream_b = cv.take<uint8_t>(total);
    uint64_t* d_hb = cv.take<uint64_t>(hb.size());
    uint64_t* d_gather = cv.take<uint64_t>(2 * (nf + 1));   // destuffed bytes, then RSTs, before each file
    const Chunks ck{d_hb, d_hb + nf + 1, d_hb + 2 * nf + 1, nf};
    ZB_CUDA(cudaMemsetAsync(stream_b, 0, total, s));
    std::vector<uint64_t> hg(2 * (nf + 1), 0);
    if (chunks) {
        ZB_CUDA(cudaMemcpyAsync(d_hb, hb.data(), hb.size() * 8, cudaMemcpyHostToDevice, s));
        dec_destuff_count<<<div_up(chunks, kThreads), kThreads, 0, s>>>(raw, ck, kept, rsts);
        ZB_LAUNCHED();
        if ((rc = scan(kept, chunks, part, koff, s)) || (rc = scan(rsts, chunks, part, roff, s))) return rc;
        dec_destuff_scatter<<<div_up(chunks, kThreads), kThreads, 0, s>>>(raw, ck, koff, roff, stream_b, rst_at);
        ZB_LAUNCHED();
        dec_pick<<<div_up(nf + 1, kThreads), kThreads, 0, s>>>(d_hb, nf + 1, koff, d_gather);
        ZB_LAUNCHED();
        dec_pick<<<div_up(nf + 1, kThreads), kThreads, 0, s>>>(d_hb, nf + 1, roff, d_gather + nf + 1);
        ZB_LAUNCHED();
        ZB_CUDA(cudaMemcpyAsync(hg.data(), d_gather, hg.size() * 8, cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
    }
    const uint32_t* words = (const uint32_t*)stream_b;

    // 3. each file's place in the batch: its stream, its intervals, its blocks
    std::vector<Geo> gb(nf);
    std::vector<Tables> tb(nf);
    std::vector<uint16_t> qb(nf * 3 * 64);
    std::vector<uint64_t> hc(3 * (nf + 1));   // first interval of each file (nf + 1), first DC slot (nf + 1), events (nf)
    uint64_t nint = 0, nblk_all = 0, total_all = 0;
    for (uint64_t f = 0; f < nf; ++f) {
        const Job& jb = jobs[plan[f]];
        Geo& g = gb[f] = geos[plan[f]];
        tb[f] = tabs[plan[f]];
        std::memcpy(&qb[f * 3 * 64], &qts[(uint64_t)plan[f] * 3 * 64], 3 * 64 * 2);
        const uint64_t nb = hg[f + 1] - hg[f], nrst = hg[nf + 2 + f] - hg[nf + 1 + f];
        const uint64_t mcus = g.total / g.bpm;
        const uint64_t need = jb.restart ? (mcus + jb.restart - 1) / jb.restart : 1;
        g.nint = need < nrst + 1 ? need : nrst + 1;
        // a missing RST ends the decode at the first block of the interval it would start
        hc[2 * (nf + 1) + f] = g.nint < need ? (g.nint * g.rblocks) << 32 : ~0ull;
        g.bit0 = jb.off * 8;
        g.bitend = (jb.off + nb) * 8;
        g.rst0 = hg[nf + 1 + f];
        g.ibase = hc[f] = nint;
        g.coef0 = nblk_all;
        g.dc0 = hc[nf + 1 + f] = total_all;
        nint += g.nint;
        nblk_all += (uint64_t)g.ncomp * g.nblk;
        total_all += g.total;
    }
    hc[nf] = nint;
    hc[2 * nf + 1] = total_all;
    Scratch meta;
    const uint64_t itiles = (nint + kScanTile - 1) / kScanTile + 1;
    if ((rc = meta.alloc(nf * (sizeof(Geo) + sizeof(Tables) + 3 * 64 * 2) + hc.size() * 8 + 8 + nint * (8 + 8 + 4 + 4) + (nint + 1) * 8 +
                             itiles * 8 + (nf + 1) * 8 + 16 * 256,
                         s)))
        return rc;
    Carve cm{meta.as<char>()};
    Geo* d_geo = cm.take<Geo>(nf);
    Tables* d_tab = cm.take<Tables>(nf);
    uint16_t* d_qt = cm.take<uint16_t>(nf * 3 * 64);
    uint64_t* d_hc = cm.take<uint64_t>(hc.size());
    int* flag = cm.take<int>(2);
    uint64_t* ia = cm.take<uint64_t>(nint);
    uint64_t* ib = cm.take<uint64_t>(nint);
    uint32_t* icnt = cm.take<uint32_t>(nint);
    int* iv_changed = cm.take<int>(nint);
    uint64_t* ifirst = cm.take<uint64_t>(nint + 1);
    uint64_t* ipart = cm.take<uint64_t>(itiles);
    uint64_t* d_sfirst = cm.take<uint64_t>(nf + 1);
    const uint64_t* d_ibase = d_hc;
    const uint64_t* d_dfirst = d_hc + nf + 1;
    unsigned long long* d_event = (unsigned long long*)(d_hc + 2 * (nf + 1));
    ZB_CUDA(cudaMemcpyAsync(d_geo, gb.data(), nf * sizeof(Geo), cudaMemcpyHostToDevice, s));
    ZB_CUDA(cudaMemcpyAsync(d_tab, tb.data(), nf * sizeof(Tables), cudaMemcpyHostToDevice, s));
    ZB_CUDA(cudaMemcpyAsync(d_qt, qb.data(), qb.size() * 2, cudaMemcpyHostToDevice, s));
    ZB_CUDA(cudaMemcpyAsync(d_hc, hc.data(), hc.size() * 8, cudaMemcpyHostToDevice, s));

    // 4. intervals and subsequences, numbered over the batch
    dec_iv_fill<<<div_up(nint, kThreads), kThreads, 0, s>>>(d_geo, d_ibase, nf, rst_at, ia, ib, icnt);
    ZB_LAUNCHED();
    if ((rc = scan(icnt, nint, ipart, ifirst, s))) return rc;
    dec_pick<<<div_up(nf + 1, kThreads), kThreads, 0, s>>>(d_ibase, nf + 1, ifirst, d_sfirst);
    ZB_LAUNCHED();
    std::vector<uint64_t> sfirst(nf + 1);   // each file's first subsequence, and the total
    ZB_CUDA(cudaMemcpyAsync(sfirst.data(), d_sfirst, (nf + 1) * 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));
    const uint64_t nsub = sfirst[nf];
    // CTAs of one file each: over its subsequences, and over its intervals
    std::vector<Cta> hcta;
    for (uint64_t f = 0; f < nf; ++f)
        for (uint64_t j = sfirst[f]; j < sfirst[f + 1]; j += kThreads) hcta.push_back({j, std::min(j + kThreads, sfirst[f + 1]), f});
    const uint64_t sctas = hcta.size();
    for (uint64_t f = 0; f < nf; ++f)
        for (uint64_t i = hc[f]; i < hc[f + 1]; i += kThreads) hcta.push_back({i, std::min(i + kThreads, hc[f + 1]), f});
    const uint64_t ictas = hcta.size() - sctas;

    Scratch sub;
    const uint64_t stiles = (nsub + kScanTile - 1) / kScanTile + 1;
    if ((rc = sub.alloc(nsub * (8 + 8 + 4 + 3 * sizeof(St) + 4 + 4) + (nsub + 1) * 8 + stiles * 8 + hcta.size() * sizeof(Cta) + 16 * 256, s))) return rc;
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
    Cta* d_cta = cs.take<Cta>(hcta.size());
    ZB_CUDA(cudaMemcpyAsync(d_cta, hcta.data(), hcta.size() * sizeof(Cta), cudaMemcpyHostToDevice, s));
    dec_sub_fill<<<div_up(nsub, kThreads), kThreads, 0, s>>>(nint, nsub, ia, ib, ifirst, send, siv, sa);
    ZB_LAUNCHED();
    const Pool P{d_tab, d_geo, d_cta, words, send, siv, ifirst};
    Pool Piv = P;
    Piv.ctas = d_cta + sctas;

    // 5. synchronisation rounds over the whole pool; flag[0]: some state of some file changed
    int changed = 1, rounds = 0;
    ZB_CUDA(cudaMemsetAsync(iv_changed, 0, nint * 4, s));
    while (changed && rounds < kMaxRounds) {
        ZB_CUDA(cudaMemsetAsync(flag, 0, 4, s));
        if (rounds + 1 == kMaxRounds) ZB_CUDA(cudaMemsetAsync(iv_changed, 0, nint * 4, s));
        ZB_CUDA(cudaMemsetAsync(owner, 0xFF, nsub * 4, s));
        dec_sync<0><<<(unsigned)sctas, kThreads, 0, s>>>(P, sa, sb, sown, owner, cnt, flag, iv_changed);
        ZB_LAUNCHED();
        dec_sync<1><<<(unsigned)sctas, kThreads, 0, s>>>(P, sa, sb, sown, owner, cnt, flag, iv_changed);
        ZB_LAUNCHED();
        ZB_CUDA(cudaMemcpyAsync(&changed, flag, 4, cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        St* t = sa;
        sa = sb;
        sb = t;
        ++rounds;
    }
    if (changed) {   // no fixed point: walk the intervals that still changed, one thread each
        dec_serial<<<(unsigned)ictas, kThreads, 0, s>>>(Piv, sb, sown, sa, cnt, iv_changed);
        ZB_LAUNCHED();
    }

    // 6. first block of each subsequence; the exact decode into zeroed storage
    if ((rc = scan(cnt, nsub, spart, boff, s))) return rc;
    std::vector<uint2> ht;   // reconstruction tiles (file, unit row), grouped by (layout, pixel format)
    struct Group { int lay, fmt; uint32_t first, count, max_unit_cols; };
    std::vector<Group> groups;
    for (int lay = 0; lay < 5; ++lay)
        for (int fmt = 0; fmt < 5; ++fmt) {
            Group gr{lay, fmt, (uint32_t)ht.size(), 0, 0};
            for (uint64_t f = 0; f < nf; ++f) {
                const Job& jb = jobs[plan[f]];
                if (jb.lay != lay || pixfmt[jb.i] != fmt) continue;
                const Geo& g = gb[f];
                gr.max_unit_cols = std::max(gr.max_unit_cols, (g.bw + kLayH[lay] - 1) / kLayH[lay]);
                const uint32_t unit_rows = (g.bh + kLayV[lay] - 1) / kLayV[lay];
                for (uint32_t y = 0; y < unit_rows; ++y) ht.push_back(make_uint2((uint32_t)f, y));
            }
            gr.count = (uint32_t)ht.size() - gr.first;
            if (gr.count) groups.push_back(gr);
        }
    Scratch blk;
    const uint64_t dtiles = (total_all + kScanTile - 1) / kScanTile + 1;
    if ((rc = blk.alloc(nblk_all * 128 + nblk_all * 4 + total_all * 4 + (total_all + 1) * 8 + dtiles * 8 + ht.size() * 8 + 16 * 256, s))) return rc;
    Carve cb{blk.as<char>()};
    int16_t* coef = cb.take<int16_t>(nblk_all * 64);
    int32_t* dcval = cb.take<int32_t>(nblk_all);
    int32_t* dcdiff = cb.take<int32_t>(total_all);
    uint64_t* pre = cb.take<uint64_t>(total_all + 1);
    uint64_t* dpart = cb.take<uint64_t>(dtiles);
    uint2* d_tiles = cb.take<uint2>(ht.size());
    ZB_CUDA(cudaMemsetAsync(coef, 0, nblk_all * 128, s));
    ZB_CUDA(cudaMemsetAsync(dcval, 0, nblk_all * 4, s));   // the MCU-padding blocks are never decoded but are read by dec_recon
    ZB_CUDA(cudaMemsetAsync(dcdiff, 0, total_all * 4, s));
    dec_final<<<(unsigned)sctas, kThreads, 0, s>>>(P, sa, boff, coef, dcdiff, d_event);
    ZB_LAUNCHED();

    // 7. DC values (each file's truncation point comes from its event slot on the device)
    if ((rc = scan((const uint32_t*)dcdiff, total_all, dpart, pre, s))) return rc;
    dec_dc<<<div_up(total_all, kThreads), kThreads, 0, s>>>(d_geo, d_dfirst, nf, dcdiff, pre, d_event, dcval, coef);
    ZB_LAUNCHED();

    // 8. reconstruction: one launch per (layout, pixel format) present
    ZB_CUDA(cudaMemcpyAsync(d_tiles, ht.data(), ht.size() * 8, cudaMemcpyHostToDevice, s));
    for (const Group& gr : groups) {
        const Recon r{d_geo, d_tiles + gr.first, gr.count, gr.max_unit_cols, coef, dcval, d_qt, d_event};
        if ((rc = launch_recon(gr.lay, gr.fmt, r, s))) return rc;
    }
    std::vector<uint64_t> ev(nf);
    ZB_CUDA(cudaMemcpyAsync(ev.data(), d_event, nf * 8, cudaMemcpyDeviceToHost, s));
    ZB_CUDA(cudaStreamSynchronize(s));   // the host arrays above are on this frame
    for (uint64_t f = 0; f < nf; ++f) status[jobs[plan[f]].i] = failed(ev[f]) ? kBad : ZB_OK;
    for (const Group& gr : groups)   // the variant of the last launch that wrote an image
        for (uint32_t t = gr.first; t < gr.first + gr.count; ++t)
            if (!failed(ev[ht[t].x])) {
                t_last_kernel = kernel_name(gr.lay, gr.fmt);
                break;
            }
    return ZB_OK;
}

extern "C" int zb_jpeg_decode(const uint8_t* data, uint64_t len, const zb_jpeg_limits* limits, zb_image* dst, int pixfmt, zb_stream stream) {
    if (!dst || (!data && len)) return ZB_ERR_INVALID_ARGUMENT;
    int status = ZB_OK;
    const int rc = zb_jpeg_decode_batch(1, &data, &len, limits, dst, &pixfmt, &status, stream);
    return rc ? rc : status;
}
