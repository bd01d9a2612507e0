// zo_jpeg_decode.cpp -- CPU oracle of the baseline JPEG decoder: jpeg.loadFromBytes (codecs/jpeg.zig:2825-2851) for SOF0 streams,
// i.e. decode (:2035-2157) with parseSOF / parseDHT / parseDQT / parseSOS / parseDRI (:1311-1644), findScanEnd (:1955-1978), the
// BitReader (:1660-1736), readCode / readMagnitudeCoded / decodeAC / decodeBlockBaseline (:1206-1308, :1933-1951), performBlockScan
// (:2397-2479), dequantizeAllBlocks, the stb integer IDCT with its level shift (:2203-2515), ycbcrToRgbAllBlocks (:2518-2749) with
// ycbcrToRgb(u8) (color.zig:1057-1068), renderRgbBlocksToPixels (:2752-2782); and getInfo (:77-180).
// TEST INFRASTRUCTURE ONLY (see zignal_oracle.h).  One thread, the reference's loops in the reference's order.
//
// Output is the native image (u8 for one component, Rgb(u8) for three); the binding (tests/jpeg_decode_oracle.py) applies
// image.convert(T) with the main oracle's zo_convert, as loadFromBytes does.
//
// Two deliberate departures, both documented in DESIGN.md §7:
//   * progressive frames (SOF2) are refused with UnsupportedProgressive once their SOF parses;
//   * restart intervals realign to the byte after the i-th RST marker (T.81 F.2.2.5) instead of discarding the bit buffer
//     (flushBits, :2431).  literal_flush = 1 restates the reference's flush exactly; only the divergence test uses it.
// Arithmetic on i32 wraps here (the reference traps on overflow in safe builds and is undefined otherwise).
// Built on its own into oracle/libzo_jpeg_decode.so (Makefile).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

extern "C" {
// jpeg.DecodeLimits (:19-33); zero disables a limit.
struct zo_jpeg_limits {
    uint64_t max_jpeg_bytes, max_marker_bytes;
    uint32_t max_width, max_height;
    uint64_t max_pixels, max_blocks, max_scans;
};
struct zo_jpeg_header {
    uint32_t width, height;
    int32_t frame_type;     // 0 baseline, 1 progressive
    int32_t num_components, precision;
    int32_t subsampling;    // -1 null, 0 444, 1 422, 2 420
};
int zo_jpeg_info(const uint8_t* data, uint64_t len, const zo_jpeg_limits* limits, zo_jpeg_header* out, char* err, int errcap);
int zo_jpeg_decode(const uint8_t* data, uint64_t len, const zo_jpeg_limits* limits, int literal_flush, uint8_t* out, uint64_t cap,
                   uint32_t* rows, uint32_t* cols, int* channels, char* err, int errcap);
int zo_jpeg_decode_coefficients(const uint8_t* data, uint64_t len, const zo_jpeg_limits* limits, int literal_flush, int32_t* coefs,
                                uint64_t cap_blocks, uint64_t* n_blocks, uint32_t* geometry, char* err, int errcap);
}

namespace {

constexpr int kUnsupported = 3, kOutOfMemory = 6, kImageTooLarge = 30, kInvalidJpeg = 31;

const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Err { const char* name; };
[[noreturn]] void fail(const char* name) { throw Err{name}; }

int status_of(const char* name) {
    if (!std::strncmp(name, "Unsupported", 11)) return kUnsupported;
    if (!std::strcmp(name, "ImageTooLarge") || !std::strcmp(name, "JpegDataTooLarge") || !std::strcmp(name, "MarkerDataLimitExceeded") ||
        !std::strcmp(name, "BlockMemoryLimitExceeded"))
        return kImageTooLarge;
    if (!std::strcmp(name, "OutOfMemory")) return kOutOfMemory;
    return kInvalidJpeg;
}
int report(const char* name, char* err, int errcap) {
    if (err && errcap > 0) {
        std::strncpy(err, name, (size_t)errcap - 1);
        err[errcap - 1] = 0;
    }
    return status_of(name);
}

zo_jpeg_limits defaults() { return {100ull << 20, 100ull << 20, 8192, 8192, 67108864ull, 1048576ull, 64}; }
bool exceeds(uint64_t limit, uint64_t v) { return limit != 0 && v > limit; }

struct Table {
    uint8_t fast[512];
    uint8_t fsize[512];
    int32_t maxcode[17];
    uint16_t mincode[17], valptr[17];
    uint8_t huffval[256];
};
struct Component { uint8_t id, h, v, tq; };
struct ScanComp { uint8_t id, td, ta; };

// BitReader (:1660-1736), plus the realignment of the T.81 restart.
struct BitReader {
    const uint8_t* data = nullptr;
    size_t len = 0, pos = 0;
    uint64_t buf = 0;
    int count = 0;
    bool fill(int n) {   // false: UnexpectedEndOfData
        while (count <= 56 && count < n) {
            if (pos >= len) return false;
            uint64_t b = data[pos++];
            if (b == 0xFF) {
                for (;;) {
                    if (pos >= len) return false;
                    const uint8_t nx = data[pos++];
                    if (nx == 0x00) break;
                    if (nx == 0xFF) continue;
                    if (nx >= 0xD0 && nx <= 0xD7) {
                        if (pos >= len) return false;
                        b = data[pos++];
                        if (b == 0xFF) continue;
                        break;
                    }
                    pos -= 2;
                    return false;
                }
            }
            buf |= b << (56 - count);
            count += 8;
        }
        return true;
    }
    bool peek(int n, uint32_t* v) {
        if (n == 0) { *v = 0; return true; }
        if (!fill(n)) return false;
        *v = (uint32_t)(buf >> (64 - n));
        return true;
    }
    void consume(int n) {
        if (n == 0) return;
        buf <<= n;
        count -= n;
    }
};

struct Eof {};   // error.UnexpectedEndOfData inside the scan

struct State {
    uint32_t width = 0, height = 0;
    int ncomp = 0;
    bool progressive = false, have_sof = false;
    Component comps[4] = {};
    bool have_dc[4] = {}, have_ac[4] = {}, have_q[4] = {};
    Table dc[4], ac[4];
    uint16_t q[4][64] = {};
    std::vector<ScanComp> scan;
    uint16_t restart_interval = 0;
    uint32_t bw = 0, bh = 0, bwa = 0, bha = 0;
    std::vector<int32_t> blocks;   // [bwa * bha][4][64]
    BitReader br;
    std::vector<size_t> rst_next;  // raw offset (in the scan) of the byte after each RST marker
    int literal = 0;

    uint8_t read_code(const Table& t) {   // readCode (:1206-1245)
        uint32_t fi = 0;
        if (!br.peek(9, &fi)) fi = 0;
        if (br.count >= 9) {
            const uint8_t v = t.fast[fi];
            if (v != 255) {
                br.consume(t.fsize[fi]);
                return v;
            }
        }
        uint32_t code = 0;
        int length = 0;
        if (br.count >= 9) {
            br.consume(9);
            code = fi;
            length = 9;
        }
        while (length < 16) {
            uint32_t bit;
            if (!br.peek(1, &bit)) throw Eof{};
            br.consume(1);
            code = (code << 1) | bit;
            ++length;
            if ((int32_t)code <= t.maxcode[length]) return t.huffval[t.valptr[length] + code - t.mincode[length]];
        }
        fail("InvalidHuffmanCode");
    }
    int32_t read_magnitude(int s) {   // readMagnitudeCoded (:1248-1260)
        if (s == 0) return 0;
        uint32_t c;
        if (!br.peek(s, &c)) throw Eof{};
        br.consume(s);
        int32_t v = (int32_t)c;
        if (v < (1 << (s - 1))) v -= (1 << s) - 1;
        return v;
    }
    void decode_block(const ScanComp& sc, int32_t* block, int32_t* pred) {   // decodeBlockBaseline (:1933-1951), decodeAC (:1263-1308)
        std::memset(block, 0, 64 * sizeof(int32_t));
        if (sc.td > 3 || !have_dc[sc.td]) fail("MissingHuffmanTable");
        const uint8_t sym = read_code(dc[sc.td]);
        if (sym > 11) fail("InvalidDCCoefficient");
        const int32_t diff = read_magnitude(sym);
        *pred = (int32_t)((uint32_t)*pred + (uint32_t)diff);
        block[0] = *pred;
        if (sc.ta > 3 || !have_ac[sc.ta]) fail("MissingHuffmanTable");
        const Table& t = ac[sc.ta];
        int k = 1;
        while (k < 64) {
            const uint8_t s = read_code(t);
            if (s == 0) return;
            const int run = s >> 4, size = s & 15;
            if (size == 0) {
                if (run != 15) fail("InvalidACCoefficient");
                k = std::min(64, k + 16);
            } else {
                k += run;
                if (k >= 64) break;
                block[kZigzag[k]] = read_magnitude(size);
                ++k;
            }
        }
    }
    // performBlockScan (:2397-2479)
    void block_scan() {
        int maxh = 1, maxv = 1;
        for (int i = 0; i < ncomp; ++i) {
            maxh = std::max<int>(maxh, comps[i].h);
            maxv = std::max<int>(maxv, comps[i].v);
        }
        const bool nonint = scan.size() == 1 && scan[0].id == 1;
        const int ys = nonint ? 1 : maxv, xs = nonint ? 1 : maxh;
        int32_t pred[4] = {0, 0, 0, 0};
        uint32_t since = 0;
        size_t interval = 0;
        int32_t tmp[64];
        try {
            for (uint32_t y = 0; y < bh; y += ys)
                for (uint32_t x = 0; x < bw; x += xs) {
                    if (restart_interval != 0 && since == restart_interval) {
                        pred[0] = pred[1] = pred[2] = pred[3] = 0;
                        since = 0;
                        br.buf = 0;
                        br.count = 0;
                        if (!literal) {   // T.81: the interval starts at the byte after its RST marker
                            if (interval >= rst_next.size()) return;
                            br.pos = rst_next[interval];
                        }
                        ++interval;
                    }
                    for (const ScanComp& sc : scan) {
                        int ci = -1;
                        for (int i = 0; i < ncomp; ++i)
                            if (comps[i].id == sc.id) { ci = i; break; }
                        if (ci < 0) fail("InvalidSOS");   // the reference reads undefined sampling factors here
                        const int vm = nonint ? 1 : comps[ci].v, hm = nonint ? 1 : comps[ci].h;
                        for (int v = 0; v < vm; ++v)
                            for (int h = 0; h < hm; ++h) {
                                const uint32_t ax = x + h, ay = y + v;
                                int32_t* b = (ay < bh && ax < bw) ? &blocks[((size_t)ay * bwa + ax) * 256 + ci * 64] : tmp;
                                br.fill(24);
                                decode_block(sc, b, &pred[ci]);
                            }
                    }
                    ++since;
                }
        } catch (Eof&) {
        }
    }
};

uint16_t be16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }

void parse_sof(State& st, const uint8_t* d, size_t n, bool progressive, const zo_jpeg_limits& lim) {   // :1311-1442
    if (st.have_sof) fail("DuplicateSOF");
    st.progressive = progressive;
    if (n < 6) fail("InvalidSOF");
    if (d[0] == 12) fail("Unsupported12BitPrecision");
    if (d[0] == 16) fail("Unsupported16BitPrecision");
    if (d[0] != 8) fail("UnsupportedPrecision");
    st.height = be16(d + 1);
    st.width = be16(d + 3);
    st.ncomp = d[5];
    if (st.width == 0 || st.height == 0) fail("InvalidSOF");
    if (exceeds(lim.max_width, st.width) || exceeds(lim.max_height, st.height)) fail("ImageTooLarge");
    if (st.ncomp == 4) fail("UnsupportedComponentCount");
    if (st.ncomp != 1 && st.ncomp != 3) fail("InvalidComponentCount");
    size_t pos = 6;
    int maxh = 0, maxv = 0;
    for (int i = 0; i < st.ncomp; ++i) {
        if (pos + 3 > n) fail("InvalidSOF");
        st.comps[i] = {d[pos], (uint8_t)(d[pos + 1] >> 4), (uint8_t)(d[pos + 1] & 15), d[pos + 2]};
        maxh = std::max<int>(maxh, st.comps[i].h);
        maxv = std::max<int>(maxv, st.comps[i].v);
        pos += 3;
    }
    if (maxh > 4 || maxv > 4) fail("UnsupportedSamplingFactor");
    if (st.ncomp == 3) {
        const Component &y = st.comps[0], &cb = st.comps[1], &cr = st.comps[2];
        if (cb.h != cr.h || cb.v != cr.v) fail("InvalidComponentCount");
        const bool c11 = cb.h == 1 && cb.v == 1;
        const bool ok = c11 && ((y.h == 1 && y.v == 1) || (y.h == 2 && y.v == 2) || (y.h == 2 && y.v == 1) || (y.h == 4 && y.v == 1));
        if (!ok) fail("UnsupportedSamplingFactor");
    }
    // maxh / maxv may be 0 for a gray component with zero sampling factors: the reference then divides by zero; refuse it
    if (maxh == 0 || maxv == 0) fail("InvalidSOF");
    const uint64_t mw = 8u * maxh, mh = 8u * maxv;
    const uint64_t wa = (st.width + mw - 1) / mw * mw, ha = (st.height + mh - 1) / mh * mh;
    st.bw = (st.width + 7) / 8;
    st.bh = (st.height + 7) / 8;
    st.bwa = (uint32_t)((wa + 7) / 8);
    st.bha = (uint32_t)((ha + 7) / 8);
    const uint64_t px = wa * ha;
    if (exceeds(lim.max_pixels, px)) fail("ImageTooLarge");
    if (exceeds(lim.max_blocks, px / 64)) fail("BlockMemoryLimitExceeded");
    st.blocks.assign((size_t)(px / 64) * 256, 0);
    st.have_sof = true;
}

void parse_dht(State& st, const uint8_t* d, size_t n) {   // :1445-1538
    if (n == 0) fail("InvalidDHT");
    size_t pos = 0;
    while (pos < n) {
        if (pos + 17 > n) fail("InvalidDHT");
        const int cls = (d[pos] >> 4) & 1, id = d[pos] & 3;
        ++pos;
        const uint8_t* bits = d + pos;
        pos += 16;
        int total = 0;
        for (int i = 0; i < 16; ++i) total += bits[i];
        if (total > 256) fail("InvalidHuffmanTable");
        if (pos + total > n) fail("InvalidDHT");
        Table t;
        std::memset(t.huffval, 0, sizeof t.huffval);
        std::memcpy(t.huffval, d + pos, (size_t)total);
        pos += total;
        std::memset(t.fast, 255, sizeof t.fast);
        std::memset(t.fsize, 0, sizeof t.fsize);
        for (int i = 0; i < 17; ++i) { t.maxcode[i] = -1; t.mincode[i] = 0; t.valptr[i] = 0; }
        uint32_t code = 0;
        int vi = 0;
        for (int i = 0; i < 16; ++i) {
            const int len = i + 1;
            if (bits[i]) {
                t.valptr[len] = (uint16_t)vi;
                t.mincode[len] = (uint16_t)code;
            }
            for (int j = 0; j < bits[i]; ++j) {
                if (code == (1u << (i + 1)) - 1) fail("InvalidHuffmanTable");
                const uint8_t sym = t.huffval[vi++];
                if (len <= 9) {
                    const uint32_t first = code << (9 - len), cnt = 1u << (9 - len);
                    for (uint32_t k = 0; k < cnt; ++k) {
                        t.fast[first + k] = sym;
                        t.fsize[first + k] = (uint8_t)len;
                    }
                }
                ++code;
            }
            if (bits[i]) t.maxcode[len] = (int32_t)code - 1;
            code <<= 1;
        }
        if (cls == 0) { st.dc[id] = t; st.have_dc[id] = true; }
        else { st.ac[id] = t; st.have_ac[id] = true; }
    }
}

void parse_dqt(State& st, const uint8_t* d, size_t n) {   // :1541-1579
    if (n == 0) fail("InvalidDQT");
    size_t pos = 0;
    while (pos < n) {
        const int prec = (d[pos] >> 4) & 15, id = d[pos] & 3;
        ++pos;
        const size_t es = prec == 0 ? 1 : 2;
        if (pos + 64 * es > n) fail("InvalidDQT");
        for (int i = 0; i < 64; ++i) st.q[id][kZigzag[i]] = es == 1 ? d[pos + i] : be16(d + pos + 2 * i);
        pos += 64 * es;
        st.have_q[id] = true;
    }
}

void parse_sos(State& st, const uint8_t* d, size_t n) {   // :1582-1637, baseline
    if (n < 6) fail("InvalidSOS");
    const int nc = d[0];
    if (nc != st.ncomp) fail("InvalidSOS");
    size_t pos = 1;
    st.scan.clear();
    for (int i = 0; i < nc; ++i) {
        if (pos + 2 > n) fail("InvalidSOS");
        st.scan.push_back({d[pos], (uint8_t)(d[pos + 1] >> 4), (uint8_t)(d[pos + 1] & 15)});
        pos += 2;
    }
    if (pos + 3 > n) fail("InvalidSOS");
    if (d[pos] != 0 || d[pos + 1] != 63 || d[pos + 2] != 0) fail("InvalidSOS");
    // a component named twice: the reference decodes it twice per MCU; this port refuses it (DESIGN.md §7)
    for (size_t i = 0; i < st.scan.size(); ++i)
        for (size_t j = i + 1; j < st.scan.size(); ++j)
            if (st.scan[i].id == st.scan[j].id) fail("InvalidSOS");
}

size_t find_scan_end(const uint8_t* d, size_t len, size_t start) {   // :1955-1978
    size_t e = start;
    while (e < len - 1) {
        if (d[e] == 0xFF) {
            const uint8_t nx = d[e + 1];
            if (nx == 0x00 || (nx >= 0xD0 && nx <= 0xD7)) {
                e += 2;
                continue;
            }
            break;
        }
        ++e;
    }
    return e;
}

void marker_payload(const uint8_t* d, size_t len, size_t& pos, uint64_t& total, const zo_jpeg_limits& lim, const uint8_t** p,
                    size_t* n) {   // readMarkerPayload (:2020-2033)
    if (pos + 4 > len) fail("UnexpectedEndOfData");
    const uint16_t l = be16(d + pos + 2);
    if (l < 2) fail("InvalidMarker");
    const size_t end = pos + 2 + l;
    if (end > len) fail("InvalidMarker");
    if (total + l < total || exceeds(lim.max_marker_bytes, total + l)) fail("MarkerDataLimitExceeded");
    total += l;
    *p = d + pos + 4;
    *n = end - pos - 4;
    pos = end;
}

// Marker.fromBytes (:1045-1105).  SOF5-SOF15 are not members, so decode skips them as unknown markers (the UnsupportedJpegVariant
// test of its else branch never sees them).
bool known_marker(uint8_t m) {
    return (m >= 0xC0 && m <= 0xC4) || m == 0xCC || (m >= 0xD0 && m <= 0xEF) || m == 0xFE;
}

// decode (:2035-2157) up to the first SOS of a baseline frame; then the entropy-coded slice [scan_start, scan_end).
void decode(State& st, const uint8_t* d, size_t len, const zo_jpeg_limits& lim) {
    if (len < 2 || d[0] != 0xFF || d[1] != 0xD8) fail("InvalidJpegFile");
    if (exceeds(lim.max_jpeg_bytes, len)) fail("JpegDataTooLarge");
    size_t pos = 2;
    uint64_t total = 0, scans = 0;
    while (pos < len - 1) {
        if (d[pos] != 0xFF) fail("InvalidMarker");
        const uint8_t m = d[pos + 1];
        if (!known_marker(m)) {
            pos += 2;
            if (pos + 2 > len) break;
            const uint16_t l = be16(d + pos);
            if (l < 2) fail("InvalidMarker");
            pos += l;
            continue;
        }
        const uint8_t* p;
        size_t n;
        switch (m) {
            case 0xD8: pos += 2; continue;
            case 0xD9: fail("NoScanData");
            case 0xC0: case 0xC2:
                marker_payload(d, len, pos, total, lim, &p, &n);
                parse_sof(st, p, n, m == 0xC2, lim);
                if (st.progressive) fail("UnsupportedProgressive");
                break;
            case 0xC1: fail("UnsupportedExtendedSequential");
            case 0xC3: fail("UnsupportedLosslessJpeg");
            case 0xC4:
                marker_payload(d, len, pos, total, lim, &p, &n);
                parse_dht(st, p, n);
                break;
            case 0xDB:
                marker_payload(d, len, pos, total, lim, &p, &n);
                parse_dqt(st, p, n);
                break;
            case 0xDA: {
                if (exceeds(lim.max_scans, scans + 1)) fail("NoScanData");   // a baseline frame with no scan decoded
                ++scans;
                // processScanMarker (:1987-2018)
                if (pos + 4 > len) fail("UnexpectedEndOfData");
                const uint16_t l = be16(d + pos + 2);
                if (l < 2) fail("InvalidMarker");
                const size_t end = pos + 2 + l;
                if (end > len) fail("InvalidMarker");
                parse_sos(st, d + pos + 4, end - pos - 4);
                const size_t se = find_scan_end(d, len, end);
                if (total + (se - pos) < total || exceeds(lim.max_marker_bytes, total + (se - pos))) fail("MarkerDataLimitExceeded");
                if (!st.have_sof) fail("BlockStorageNotAllocated");
                st.br.data = d + end;
                st.br.len = se - end;
                for (size_t i = 0; i + 1 < st.br.len; ++i)
                    if (st.br.data[i] == 0xFF) {
                        if (st.br.data[i + 1] >= 0xD0 && st.br.data[i + 1] <= 0xD7) st.rst_next.push_back(i + 2);
                        ++i;
                    }
                return;
            }
            case 0xDD:
                marker_payload(d, len, pos, total, lim, &p, &n);
                if (n != 2) fail("InvalidDRI");
                st.restart_interval = be16(p);
                break;
            case 0xCC: fail("UnsupportedArithmeticCoding");
            case 0xDE: fail("UnsupportedHierarchicalJpeg");
            case 0xDC: fail("UnsupportedJpegVariant");
            default: {
                if (m >= 0xC5 && m <= 0xCF) fail("UnsupportedJpegVariant");
                if (pos + 4 > len) goto done;
                const uint16_t l = be16(d + pos + 2);
                if (total + l < total || exceeds(lim.max_marker_bytes, total + l)) fail("MarkerDataLimitExceeded");
                total += l;
                pos += 2 + (size_t)l;
            }
        }
    }
done:
    fail("NoScanData");
}

// stb's integer IDCT (:2203-2313) with the level shift of component 0 (:2498-2515); u32 arithmetic so overflow wraps.
#define F2F(x) ((int32_t)std::lround((x) * 4096.0f))
void idct1d(const int32_t* s, int32_t* o) {
    auto M = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); };
    auto A = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); };
    auto S = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); };
    int32_t p2 = s[2], p3 = s[6];
    int32_t p1 = M(A(p2, p3), F2F(0.5411961f));
    int32_t t2 = A(p1, M(p3, F2F(-1.847759065f)));
    int32_t t3 = A(p1, M(p2, F2F(0.765366865f)));
    p2 = s[0];
    p3 = s[4];
    int32_t t0 = M(A(p2, p3), 4096), t1 = M(S(p2, p3), 4096);
    const int32_t x0 = A(t0, t3), x3 = S(t0, t3), x1 = A(t1, t2), x2 = S(t1, t2);
    t0 = s[7]; t1 = s[5]; t2 = s[3]; t3 = s[1];
    p3 = A(t0, t2);
    int32_t p4 = A(t1, t3);
    p1 = A(t0, t3);
    p2 = A(t1, t2);
    const int32_t p5 = M(A(p3, p4), F2F(1.175875602f));
    t0 = M(t0, F2F(0.298631336f));
    t1 = M(t1, F2F(2.053119869f));
    t2 = M(t2, F2F(3.072711026f));
    t3 = M(t3, F2F(1.501321110f));
    p1 = A(p5, M(p1, F2F(-0.899976223f)));
    p2 = A(p5, M(p2, F2F(-2.562915447f)));
    p3 = M(p3, F2F(-1.961570560f));
    p4 = M(p4, F2F(-0.390180644f));
    t3 = A(t3, A(p1, p4));
    t2 = A(t2, A(p2, p3));
    t1 = A(t1, A(p2, p4));
    t0 = A(t0, A(p1, p3));
    o[0] = x0; o[1] = x1; o[2] = x2; o[3] = x3; o[4] = t0; o[5] = t1; o[6] = t2; o[7] = t3;
}
void idct8x8(int32_t* b) {
    bool zero = true;
    for (int i = 1; i < 64; ++i) zero = zero && b[i] == 0;
    if (zero) {
        const int32_t v = (int32_t)((uint32_t)b[0] + 4u) >> 3;
        for (int i = 0; i < 64; ++i) b[i] = v;
        return;
    }
    int32_t tmp[64];
    auto out8 = [](const int32_t* r, int32_t add, int sh, int32_t* w, int stride) {
        auto A = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); };
        auto S = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); };
        const int32_t x0 = A(r[0], add), x1 = A(r[1], add), x2 = A(r[2], add), x3 = A(r[3], add);
        w[0 * stride] = A(x0, r[7]) >> sh; w[1 * stride] = A(x1, r[6]) >> sh;
        w[2 * stride] = A(x2, r[5]) >> sh; w[3 * stride] = A(x3, r[4]) >> sh;
        w[4 * stride] = S(x3, r[4]) >> sh; w[5 * stride] = S(x2, r[5]) >> sh;
        w[6 * stride] = S(x1, r[6]) >> sh; w[7 * stride] = S(x0, r[7]) >> sh;
    };
    for (int c = 0; c < 8; ++c) {   // pass 1: down each column
        int32_t s[8], r[8];
        for (int v = 0; v < 8; ++v) s[v] = b[v * 8 + c];
        idct1d(s, r);
        out8(r, 512, 10, tmp + c, 8);
    }
    for (int y = 0; y < 8; ++y) {   // pass 2: along each row
        int32_t r[8];
        idct1d(tmp + y * 8, r);
        out8(r, 65536, 17, b + y * 8, 1);
    }
}

uint8_t clamp8(int64_t v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
void ycc_to_rgb(int32_t y, int32_t cb, int32_t cr, uint8_t* o) {   // ycbcrToRgb(u8) (color.zig:1057-1068)
    const int64_t Y = y, B = (int64_t)cb - 128, R = (int64_t)cr - 128;
    o[0] = clamp8((65536 * Y + 91881 * R + 32768) >> 16);
    o[1] = clamp8((65536 * Y - 22554 * B - 46802 * R + 32768) >> 16);
    o[2] = clamp8((65536 * Y + 116130 * B + 32768) >> 16);
}

// The native image of ycbcrToRgbAllBlocks + renderRgbBlocksToPixels.  out: rows x cols x (1 or 3) u8.
void to_pixels(State& st, uint8_t* out) {
    const int ch = st.ncomp == 1 ? 1 : 3;
    const size_t nb = (size_t)st.bwa * st.bha;
    // dequantizeAllBlocks (:2482-2495), idctAllBlocks (:2498-2515)
    for (int c = 0; c < st.ncomp; ++c)
        if (st.comps[c].tq > 3 || !st.have_q[st.comps[c].tq]) fail("MissingQuantTable");
    for (size_t b = 0; b < nb; ++b)
        for (int c = 0; c < st.ncomp; ++c) {
            int32_t* blk = &st.blocks[b * 256 + c * 64];
            const uint16_t* q = st.q[st.comps[c].tq];
            for (int i = 0; i < 64; ++i) blk[i] = (int32_t)((uint32_t)blk[i] * q[i]);
            idct8x8(blk);
            if (c == 0)
                for (int i = 0; i < 64; ++i) blk[i] = (int32_t)((uint32_t)blk[i] + 128u);
        }
    auto put = [&](size_t b, int i, const uint8_t* rgb) {
        const uint32_t by = (uint32_t)(b / st.bwa), bx = (uint32_t)(b % st.bwa);
        const uint32_t py = by * 8 + i / 8, px = bx * 8 + i % 8;
        if (by >= st.bh || bx >= st.bw || py >= st.height || px >= st.width) return;
        std::memcpy(out + ((size_t)py * st.width + px) * ch, rgb, (size_t)ch);
    };
    if (st.ncomp == 1) {
        for (size_t b = 0; b < nb; ++b)
            for (int i = 0; i < 64; ++i) {
                const int32_t v = st.blocks[b * 256 + i];
                const uint8_t g = clamp8(v);
                put(b, i, &g);
            }
        return;
    }
    const int mh = st.comps[0].h, mv = st.comps[0].v;
    if (mh == 1 && mv == 1) {   // 4:4:4, 16.16 on the unclamped Y and centred chroma
        for (size_t b = 0; b < nb; ++b)
            for (int i = 0; i < 64; ++i) {
                const int32_t* s = &st.blocks[b * 256];
                const int32_t Y = s[i], Cb = s[64 + i], Cr = s[128 + i];
                auto M = [](int32_t a, int32_t k) { return (int32_t)((uint32_t)a * (uint32_t)k); };
                auto A = [](int32_t a, int32_t c) { return (int32_t)((uint32_t)a + (uint32_t)c); };
                const int32_t r = A(Y, A(M(91881, Cr), 32768) >> 16);
                const int32_t g = (int32_t)((uint32_t)Y - (uint32_t)(A(A(M(22554, Cb), M(46802, Cr)), 32768) >> 16));
                const int32_t bl = A(Y, A(M(116130, Cb), 32768) >> 16);
                const uint8_t rgb[3] = {clamp8(r), clamp8(g), clamp8(bl)};
                put(b, i, rgb);
            }
        return;
    }
    // 4:2:2, 4:1:1 and 4:2:0: f32 lerp inside the MCU's chroma block, indices clamped to [0, 7], @round half away from zero
    const float sx = mh == 4 ? 0.25f : 0.5f, sy = mv == 2 ? 0.5f : 1.0f;
    for (uint32_t my = 0; my < st.bh; my += mv)
        for (uint32_t mx = 0; mx < st.bw; mx += mh) {
            const size_t cb_idx = (size_t)my * st.bwa + mx;
            const int32_t* cbb = &st.blocks[cb_idx * 256 + 64];
            const int32_t* crb = &st.blocks[cb_idx * 256 + 128];
            for (int v = 0; v < mv; ++v)
                for (int h = 0; h < mh; ++h) {
                    if (my + v >= st.bh || mx + h >= st.bw) continue;
                    const size_t yb = (size_t)(my + v) * st.bwa + mx + h;
                    for (int i = 0; i < 64; ++i) {
                        const int py = i / 8, px = i % 8;
                        const int32_t Y = st.blocks[yb * 256 + i];
                        const float cxf = ((float)(h * 8 + px) + 0.5f) * sx - 0.5f;
                        const int cx0 = (int)std::min(std::max(std::floor(cxf), 0.0f), 7.0f), cx1 = std::min(7, cx0 + 1);
                        const float fx = cxf - (float)cx0;
                        int32_t Cb, Cr;
                        if (mv == 1) {
                            const float a = (float)cbb[py * 8 + cx0], bb = (float)cbb[py * 8 + cx1];
                            const float c = (float)crb[py * 8 + cx0], dd = (float)crb[py * 8 + cx1];
                            Cb = (int32_t)std::round(std::fma(bb - a, fx, a));
                            Cr = (int32_t)std::round(std::fma(dd - c, fx, c));
                        } else {
                            const float cyf = ((float)(v * 8 + py) + 0.5f) * sy - 0.5f;
                            const int cy0 = (int)std::min(std::max(std::floor(cyf), 0.0f), 7.0f), cy1 = std::min(7, cy0 + 1);
                            const float fy = cyf - (float)cy0;
                            auto bil = [&](const int32_t* k) {
                                const float k00 = (float)k[cy0 * 8 + cx0], k10 = (float)k[cy0 * 8 + cx1];
                                const float k01 = (float)k[cy1 * 8 + cx0], k11 = (float)k[cy1 * 8 + cx1];
                                const float i0 = std::fma(k10 - k00, fx, k00), i1 = std::fma(k11 - k01, fx, k01);
                                return (int32_t)std::round(std::fma(i1 - i0, fy, i0));
                            };
                            Cb = bil(cbb);
                            Cr = bil(crb);
                        }
                        uint8_t rgb[3];
                        ycc_to_rgb(clamp8(Y), clamp8((int64_t)Cb + 128), clamp8((int64_t)Cr + 128), rgb);
                        put(yb, i, rgb);
                    }
                }
        }
}

int run(const uint8_t* data, uint64_t len, const zo_jpeg_limits* limits, int literal, State& st, char* err, int errcap) {
    const zo_jpeg_limits lim = limits ? *limits : defaults();
    try {
        st.literal = literal;
        decode(st, data, (size_t)len, lim);
        st.block_scan();
    } catch (Err& e) {
        return report(e.name, err, errcap);
    }
    return 0;
}

}  // namespace

extern "C" int zo_jpeg_info(const uint8_t* d, uint64_t len, const zo_jpeg_limits* limits, zo_jpeg_header* out, char* err, int errcap) {
    // getInfo (:77-180) over a fixed reader: running out of bytes is error.EndOfStream
    const zo_jpeg_limits lim = limits ? *limits : defaults();
    uint64_t pos = 0, read = 0, markers = 0;
    auto take = [&](uint8_t* b) {
        if (pos >= len) throw Err{"EndOfStream"};
        *b = d[pos++];
        ++read;
    };
    try {
        uint8_t a, b;
        take(&a);
        take(&b);
        if (a != 0xFF || b != 0xD8) fail("InvalidJpegFile");
        for (;;) {
            for (;;) {
                take(&a);
                if (exceeds(lim.max_jpeg_bytes, read)) fail("ImageTooLarge");
                if (a == 0xFF) break;
            }
            take(&b);
            while (b == 0xFF) {
                take(&b);
                if (exceeds(lim.max_jpeg_bytes, read)) fail("ImageTooLarge");
            }
            if (b == 0x00) continue;
            if (++markers > 10000) fail("ImageTooLarge");
            if (b == 0x01 || (b >= 0xD0 && b <= 0xD8)) continue;
            if (b == 0xD9) fail("MissingSOF");
            uint8_t h, l;
            take(&h);
            take(&l);
            const uint32_t length = (uint32_t)(h << 8 | l);
            if (length < 2) fail("InvalidMarker");
            const bool sof = b >= 0xC0 && b <= 0xCF && b != 0xC4 && b != 0xC8 && b != 0xCC;
            if (sof) {
                const uint32_t payload = length - 2;
                if (payload < 6) fail("InvalidSOF");
                if (exceeds(lim.max_jpeg_bytes, read + payload)) fail("ImageTooLarge");
                uint8_t p[6];
                for (int i = 0; i < 6; ++i) take(&p[i]);
                out->precision = p[0];
                out->height = (uint32_t)(p[1] << 8 | p[2]);
                out->width = (uint32_t)(p[3] << 8 | p[4]);
                out->num_components = p[5];
                out->frame_type = b == 0xC2 ? 1 : 0;
                out->subsampling = -1;
                if (p[5] == 3 && payload - 6 >= 9) {
                    uint8_t f[9];
                    for (int i = 0; i < 9; ++i) take(&f[i]);
                    if (f[4] == 0x11 && f[7] == 0x11) out->subsampling = f[1] == 0x11 ? 0 : (f[1] == 0x21 ? 1 : (f[1] == 0x22 ? 2 : -1));
                }
                return 0;
            }
            const uint32_t skip = length - 2;
            if (exceeds(lim.max_jpeg_bytes, read + skip)) fail("ImageTooLarge");
            const uint64_t n = std::min<uint64_t>(skip, len - pos);
            pos += n;
            read += n;
        }
    } catch (Err& e) {
        return report(e.name, err, errcap);
    }
}

extern "C" int zo_jpeg_decode(const uint8_t* data, uint64_t len, const zo_jpeg_limits* limits, int literal_flush, uint8_t* out,
                              uint64_t cap, uint32_t* rows, uint32_t* cols, int* channels, char* err, int errcap) {
    State st;
    int rc = run(data, len, limits, literal_flush, st, err, errcap);
    if (rc) return rc;
    *rows = st.height;
    *cols = st.width;
    *channels = st.ncomp == 1 ? 1 : 3;
    const uint64_t need = (uint64_t)st.height * st.width * (uint64_t)*channels;
    if (cap < need || !out) return kOutOfMemory;
    std::memset(out, 0, need);
    try {
        to_pixels(st, out);
    } catch (Err& e) {
        return report(e.name, err, errcap);
    }
    return 0;
}

// The block storage after the scan (before dequantisation): (bwa * bha) x ncomp x 64 i32, natural order.  geometry receives
// {bw, bh, bwa, bha, ncomp}.
extern "C" int zo_jpeg_decode_coefficients(const uint8_t* data, uint64_t len, const zo_jpeg_limits* limits, int literal_flush,
                                           int32_t* coefs, uint64_t cap_blocks, uint64_t* n_blocks, uint32_t* geometry, char* err,
                                           int errcap) {
    State st;
    int rc = run(data, len, limits, literal_flush, st, err, errcap);
    if (rc) return rc;
    const uint64_t nb = (uint64_t)st.bwa * st.bha;
    *n_blocks = nb;
    if (geometry) {
        geometry[0] = st.bw; geometry[1] = st.bh; geometry[2] = st.bwa; geometry[3] = st.bha; geometry[4] = (uint32_t)st.ncomp;
    }
    if (cap_blocks < nb || !coefs) return kOutOfMemory;
    for (uint64_t b = 0; b < nb; ++b)
        for (int c = 0; c < st.ncomp; ++c) std::memcpy(coefs + (b * st.ncomp + c) * 64, &st.blocks[b * 256 + c * 64], 256);
    return 0;
}
