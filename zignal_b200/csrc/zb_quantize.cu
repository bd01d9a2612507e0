// zb_quantize.cu -- colour quantization and dithering (reference image/quantize.zig, image/dither.zig) on the device.
//
//   zb_median_cut     : quantize.zig:175-412.  The device builds the 32768-bin histogram of the 5-bit keys r>>3, g>>3, b>>3 (after
//                       convertColor to Rgb(u8)) with, per bin, its count and the raster index of its first pixel.  The host orders the
//                       touched bins by first index -- the reference's `color_list` is in first-touch order, and that order decides the
//                       cuts -- and runs the box loop exactly as the reference does, std.sort.heap included (it is unstable, so ties in
//                       the split dimension decide which colours land in which box).
//   zb_build_palette  : quantize.zig:502-527.
//   zb_color_lut      : ColorLookupTable.init, quantize.zig:66-159: one thread per entry, minimum of dist << 8 | i.
//   zb_palette_lookup : ColorLookupTable.lookup(convertColor(Rgb, px)) per pixel into a u8 index image.
//   zb_dither         : dither.apply, dither.zig:34-331.  Ordered dithering is elementwise.  Floyd-Steinberg and Atkinson run as a
//                       wavefront (below).
//
// Error diffusion as a wavefront.  Every contribution is a clamped add, clampToU8(v + divTruncPow2(err * w, shift)), so what a pixel
// holds when it is quantized is a sequence, not a sum: its contributions must arrive in the raster order of their sources.  Those are
//   Floyd-Steinberg : (r-1, c-1) * 1, (r-1, c) * 5, (r-1, c+1) * 3, (r, c-1) * 7, each / 16;
//   Atkinson        : (r-2, c), (r-1, c-1), (r-1, c), (r-1, c+1), (r, c-2), (r, c-1), each / 8;
// and the reference's fast and bounds-checked branches apply the same contributions in the same order, so a contribution is simply
// dropped when its target lies outside the image.  Pixel (r, c) is final once (r-1, c+1) and (r, c-1) are done, so row r can run two
// columns behind row r-1.
//
// One warp runs a band of 32 rows, lane i on row r0 + i, at column t - 1 - 2i in step t.  Each lane keeps a window of three pixels of the
// row below (columns c-1, c, c+1).  In step t it (1) starts the window's column c+1 from the original pixel plus, for Atkinson, the
// (r-1, c+1) error its upper neighbour produced in step t-1, (2) applies the right contributions of (r, c-2) and (r, c-1) to the value
// it was handed for (r, c), quantizes it and writes the palette colour, (3) adds the error to the window, and (4) hands column c-1 of the
// row below, which now has every contribution from above, together with its error at (r, c), to lane i+1 by shuffle.  So each pixel gets
// its contributions in raster order.  Lane 31 writes the same pair into a per-band slot array in stream-ordered scratch, and lane 0 of
// the next band reads it from there: slot[c] = {value of (r0', c-1), error at (r0'-1, c)}.
//
// Between bands a progress counter per band (release by lane 31 every `publish` columns, acquire by the whole next warp) orders the slot
// writes before their reads, and orders the upper band's reads of the original first row of the lower band before the lower band
// overwrites it.  The lower band waits in chunks of 32 columns and loads a chunk of slots with one load per lane.  Bands are claimed with
// a global ticket (four per CTA, in order), so a warp only ever waits on a band already held by a running warp; by induction over the
// band index every wait ends (DESIGN.md §4.6).  Nothing times out and nothing iterates to a fixed point.
#include <cuda/atomic>

#include <algorithm>
#include <vector>

#include "zb_convert.cuh"
#include "zb_internal.h"

namespace zb {

std::atomic<int> g_tune_dither_publish{32};

namespace {

constexpr int kLutSize = 32768;
constexpr int kTileThreads = 256;       // ordered dither / lookup: threads per CTA
constexpr int kTilePx = 8;              // pixels per thread and row
constexpr int kTileRows = 16;           // rows per CTA
constexpr int kDiffuseWarps = 4;        // bands per error-diffusion CTA
constexpr uint32_t kZeroErr = 256u | (256u << 10) | (256u << 20);

// The palette crosses the ABI as data: at most 256 x 3 bytes, zero-padded, in the kernel parameters.
struct Pal {
    uint8_t rgb[256 * 3];
};

__device__ __forceinline__ uint32_t pal_word(const Pal& p, int i) {
    return (uint32_t)p.rgb[3 * i] | ((uint32_t)p.rgb[3 * i + 1] << 8) | ((uint32_t)p.rgb[3 * i + 2] << 16);
}

// The LUT (32 KB) and the zero-padded palette as packed words, into shared memory.
__device__ __forceinline__ void load_tables(uint8_t* slut, uint32_t* spal, const uint8_t* lut, const Pal* pal) {
    if (((uintptr_t)lut & 15) == 0) {
        const uint4* src = (const uint4*)lut;
        uint4* dst = (uint4*)slut;
        for (int i = threadIdx.x; i < kLutSize / 16; i += blockDim.x) dst[i] = src[i];
    } else {   // a LUT inside a larger allocation need not be 16-byte aligned
        for (int i = threadIdx.x; i < kLutSize; i += blockDim.x) slut[i] = lut[i];
    }
    if (pal)
        for (int i = threadIdx.x; i < 256; i += blockDim.x) spal[i] = pal_word(*pal, i);
}

__device__ __forceinline__ int lut_key(int r, int g, int b) { return ((r >> 3) << 10) | ((g >> 3) << 5) | (b >> 3); }

// Pixel -> Rgb(u8) by convertColor (color.zig:108-151).
template <int SF> __device__ __forceinline__ void to_rgb8(const void* img, size_t stride, uint32_t r, uint32_t c, uint8_t* rgb) {
    using CT = typename Fmt<SF>::CT;
    const CT* p = (const CT*)img + ((size_t)r * stride + c) * Fmt<SF>::N;
    if constexpr (SF == ZB_PIX_RGB8) {
        rgb[0] = p[0]; rgb[1] = p[1]; rgb[2] = p[2];
    } else {
        convert_color<SF, ZB_PIX_RGB8>(p, rgb);
    }
}

// ---- median cut: histogram ----------------------------------------------------------------------------------------------------------
// counts[key] += 1 and first[key] = min(raster index); lanes of a warp hold consecutive pixels of one row, so equal keys in a warp
// are aggregated (__match_any_sync) and the group's lowest lane carries its smallest index.
template <int SF>
__global__ void __launch_bounds__(kTileThreads) mc_histogram(const void* img, size_t stride, uint32_t rows, uint32_t cols,
                                                             uint32_t* counts, uint32_t* first) {
    const int r = ZB_GRID_ROW();
    if ((uint32_t)r >= rows) return;
    const uint64_t c_wide = (uint64_t)blockIdx.x * kTileThreads + threadIdx.x;
    const bool in = c_wide < cols;
    const int lane = threadIdx.x & 31;
    uint32_t key = 0x10000u + lane;   // never matches a real key
    if (in) {
        uint8_t rgb[3];
        to_rgb8<SF>(img, stride, r, (uint32_t)c_wide, rgb);
        key = (uint32_t)lut_key(rgb[0], rgb[1], rgb[2]);
    }
    const unsigned group = __match_any_sync(0xffffffffu, key);
    if (in && (__ffs(group) - 1) == lane) {
        atomicAdd(counts + key, (uint32_t)__popc(group));
        atomicMin(first + key, (uint32_t)r * cols + (uint32_t)c_wide);
    }
}

// ---- ColorLookupTable.init ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) color_lut_kernel(Pal pal, uint32_t n, uint8_t* lut) {
    __shared__ uint32_t spal[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) spal[i] = pal_word(pal, i);
    __syncthreads();
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= kLutSize) return;
    const int r5 = e >> 10, g5 = (e >> 5) & 31, b5 = e & 31;
    const int tr = (r5 << 3) | (r5 >> 2), tg = (g5 << 3) | (g5 >> 2), tb = (b5 << 3) | (b5 >> 2);   // quantize.zig:84-88
    uint32_t best = 0xffffffffu;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t w = spal[i];
        const int dr = (int)(w & 255) - tr, dg = (int)((w >> 8) & 255) - tg, db = (int)(w >> 16) - tb;
        const uint32_t score = ((uint32_t)(dr * dr + dg * dg + db * db) << 8) | i;   // :139 / :152
        best = min(best, score);
    }
    lut[e] = (uint8_t)(best & 0xff);
}

// ---- elementwise passes: ordered dither and index lookup ----------------------------------------------------------------------------
// One CTA per kTileRows rows x (kTileThreads * kTilePx) columns; the LUT sits in shared memory.

__device__ __forceinline__ int clamp_u8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// dither.zig:113-196: offset (bayer[r & 7][c & 7] - 32) >> 1 on every channel, clamp, 5-bit key, palette colour.  The SIMD and scalar
// paths of the reference compute the same thing for every column (the vector path runs on 8-aligned columns, so k == c & 7).
__constant__ int8_t c_bayer[8][8] = {
    {0, 32, 8, 40, 2, 34, 10, 42},   {48, 16, 56, 24, 50, 18, 58, 26}, {12, 44, 4, 36, 14, 46, 6, 38}, {60, 28, 52, 20, 62, 30, 54, 22},
    {3, 35, 11, 43, 1, 33, 9, 41},   {51, 19, 59, 27, 49, 17, 57, 25}, {15, 47, 7, 39, 13, 45, 5, 37}, {63, 31, 55, 23, 61, 29, 53, 21},
};

__global__ void __launch_bounds__(kTileThreads) ordered_kernel(uint8_t* img, size_t stride, uint32_t rows, uint32_t cols,
                                                               const uint8_t* lut, Pal pal) {
    __shared__ __align__(16) uint8_t slut[kLutSize];
    __shared__ uint32_t spal[256];
    const int tile = ZB_GRID_ROW();
    const uint32_t r0 = (uint32_t)tile * kTileRows;
    if (r0 >= rows) return;
    load_tables(slut, spal, lut, &pal);
    __syncthreads();
    const uint64_t c0 = (uint64_t)blockIdx.x * kTileThreads * kTilePx;
    const uint32_t r1 = min(rows, r0 + kTileRows);
    for (uint32_t r = r0; r < r1; ++r) {
        uint8_t* row = img + (size_t)r * stride * 3;
        int off[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) off[k] = ((int)c_bayer[r & 7][k] - 32) >> 1;
#pragma unroll
        for (int k = 0; k < kTilePx; ++k) {
            const uint64_t c = c0 + (uint64_t)k * kTileThreads + threadIdx.x;
            if (c >= cols) break;
            uint8_t* p = row + c * 3;
            const int o = off[c & 7];
            const int key = lut_key(clamp_u8(p[0] + o), clamp_u8(p[1] + o), clamp_u8(p[2] + o));
            const uint32_t q = spal[slut[key]];
            p[0] = (uint8_t)q;
            p[1] = (uint8_t)(q >> 8);
            p[2] = (uint8_t)(q >> 16);
        }
    }
}

template <int SF>
__global__ void __launch_bounds__(kTileThreads) lookup_kernel(const void* src, size_t src_stride, uint8_t* dst, size_t dst_stride,
                                                              uint32_t rows, uint32_t cols, const uint8_t* lut) {
    __shared__ __align__(16) uint8_t slut[kLutSize];
    const int tile = ZB_GRID_ROW();
    const uint32_t r0 = (uint32_t)tile * kTileRows;
    if (r0 >= rows) return;
    load_tables(slut, nullptr, lut, nullptr);
    __syncthreads();
    const uint64_t c0 = (uint64_t)blockIdx.x * kTileThreads * kTilePx;
    const uint32_t r1 = min(rows, r0 + kTileRows);
    for (uint32_t r = r0; r < r1; ++r) {
#pragma unroll
        for (int k = 0; k < kTilePx; ++k) {
            const uint64_t c = c0 + (uint64_t)k * kTileThreads + threadIdx.x;
            if (c >= cols) break;
            uint8_t rgb[3];
            to_rgb8<SF>(src, src_stride, r, (uint32_t)c, rgb);
            dst[(size_t)r * dst_stride + c] = slut[lut_key(rgb[0], rgb[1], rgb[2])];
        }
    }
}

// ---- error diffusion ----------------------------------------------------------------------------------------------------------------

struct Px { int r, g, b; };

__device__ __forceinline__ Px unpack_px(uint32_t w) { return {(int)(w & 255), (int)((w >> 8) & 255), (int)((w >> 16) & 255)}; }
__device__ __forceinline__ uint32_t pack_px(Px p) { return (uint32_t)p.r | ((uint32_t)p.g << 8) | ((uint32_t)p.b << 16); }
// errors lie in [-255, 255]: 10 bits per channel, biased by 256
__device__ __forceinline__ Px unpack_err(uint32_t w) {
    return {(int)(w & 1023) - 256, (int)((w >> 10) & 1023) - 256, (int)((w >> 20) & 1023) - 256};
}
__device__ __forceinline__ uint32_t pack_err(Px e) {
    return (uint32_t)(e.r + 256) | ((uint32_t)(e.g + 256) << 10) | ((uint32_t)(e.b + 256) << 20);
}

// dither.zig:97-104, :224-228
__device__ __forceinline__ int div_trunc_pow2(int v, int shift) { return v >= 0 ? v >> shift : (v + (1 << shift) - 1) >> shift; }
template <int W, int SHIFT> __device__ __forceinline__ void update(Px& p, Px e) {
    p.r = clamp_u8(p.r + div_trunc_pow2(e.r * W, SHIFT));
    p.g = clamp_u8(p.g + div_trunc_pow2(e.g * W, SHIFT));
    p.b = clamp_u8(p.b + div_trunc_pow2(e.b * W, SHIFT));
}

__device__ __forceinline__ uint32_t load_rgb(const uint8_t* img, size_t stride, uint32_t r, uint32_t c) {
    const uint8_t* p = img + ((size_t)r * stride + c) * 3;
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
}

struct DiffuseParams {
    uint8_t* img;
    size_t stride;
    uint32_t rows, cols;
    const uint8_t* lut;
    uint32_t* progress;   // per band: slots published (release by the band's lane 31)
    uint32_t* ticket;     // CTA tickets
    uint2* slots;         // per band: cols + 1 slots {value of (r0 + 32, c - 1), packed error at (r0 + 31, c)}
    uint32_t nbands;
    uint32_t publish;     // lane 31 publishes every `publish` columns
};

template <bool ATK>
__global__ void __launch_bounds__(32 * kDiffuseWarps) diffuse_kernel(DiffuseParams p, Pal pal) {
    __shared__ __align__(16) uint8_t slut[kLutSize];
    __shared__ uint32_t spal[256];
    __shared__ uint32_t first_band;
    load_tables(slut, spal, p.lut, &pal);
    if (threadIdx.x == 0) first_band = atomicAdd(p.ticket, 1u) * kDiffuseWarps;
    __syncthreads();
    const uint32_t band = first_band + threadIdx.x / 32;
    if (band >= p.nbands) return;   // uniform per warp
    const int lane = threadIdx.x & 31;
    const uint32_t cols = p.cols;
    const uint32_t R = band * 32 + lane;
    const bool row_ok = R < p.rows;
    const bool below_ok = R + 1 < p.rows;
    uint2* out_slots = p.slots + (size_t)band * (cols + 1);
    const uint2* in_slots = p.slots + (size_t)(band - 1) * (cols + 1);
    cuda::atomic_ref<uint32_t, cuda::thread_scope_device> upstream(p.progress[band ? band - 1 : 0]);
    uint32_t seen = 0;                    // progress of the band above known to this warp

    Px b0{0, 0, 0}, b1{0, 0, 0};          // the window on the row below: columns c-1, c
    Px e1{0, 0, 0}, e2{0, 0, 0};          // errors at (R, c-1), (R, c-2)
    uint32_t hv = 0, ea = kZeroErr;       // handed value of (R, c); error at (R-1, c+1)
    uint32_t chunk_h = 0, chunk_e = kZeroErr;
    uint32_t pf = (lane == 0 && below_ok) ? load_rgb(p.img, p.stride, R + 1, 0) : 0;   // original (R+1, c+1)
    const int64_t steps = (int64_t)cols + 64;
    for (int64_t t = 0; t < steps; ++t) {
        const int64_t c = t - 1 - 2 * lane;
        // lane 0's inputs come in chunks of 32 slots: from the band above, or for band 0 from the image's first row
        if ((t & 31) == 0 && t <= cols) {
            const uint32_t s = (uint32_t)t + lane;
            if (band == 0) {
                chunk_h = (s >= 1 && s <= cols) ? load_rgb(p.img, p.stride, 0, s - 1) : 0;
                chunk_e = kZeroErr;
            } else {
                const uint32_t need = min((uint32_t)t + 32, cols + 1);
                while (seen < need) {
                    seen = upstream.load(cuda::memory_order_acquire);
                    seen = __reduce_min_sync(0xffffffffu, seen);
                }
                const uint2 v = s <= cols ? __ldcg(in_slots + s) : make_uint2(0, kZeroErr);
                chunk_h = v.x;
                chunk_e = v.y;
            }
        }
        const uint32_t h0 = __shfl_sync(0xffffffffu, chunk_h, (int)(t & 31));
        const uint32_t e0 = __shfl_sync(0xffffffffu, chunk_e, (int)(t & 31));
        if (lane == 0) { hv = h0; ea = e0; }

        uint32_t out_h = 0, out_e = kZeroErr;
        if (row_ok && c >= -1 && c <= (int64_t)cols) {
            Px bn{0, 0, 0};
            if (below_ok && c + 1 < (int64_t)cols) {   // start column c+1 of the row below
                bn = unpack_px(pf);
                if constexpr (ATK) update<1, 3>(bn, unpack_err(ea));              // from (R-1, c+1)
            }
            if (c >= 0 && c < (int64_t)cols) {
                Px v = unpack_px(hv);
                if constexpr (ATK) {
                    update<1, 3>(v, e2);                                          // from (R, c-2)
                    update<1, 3>(v, e1);                                          // from (R, c-1)
                } else {
                    update<7, 4>(v, e1);                                          // from (R, c-1)
                }
                const uint32_t q = spal[slut[lut_key(v.r, v.g, v.b)]];
                uint8_t* dst = p.img + ((size_t)R * p.stride + (size_t)c) * 3;
                dst[0] = (uint8_t)q;
                dst[1] = (uint8_t)(q >> 8);
                dst[2] = (uint8_t)(q >> 16);
                const Px qp = unpack_px(q);
                const Px err{v.r - qp.r, v.g - qp.g, v.b - qp.b};
                if constexpr (ATK) {
                    update<1, 3>(b0, err);
                    update<1, 3>(b1, err);
                    update<1, 3>(bn, err);
                } else {
                    update<3, 4>(b0, err);
                    update<5, 4>(b1, err);
                    update<1, 4>(bn, err);
                }
                e2 = e1;
                e1 = err;
                out_e = pack_err(err);
            }
            out_h = pack_px(b0);   // column c-1 of the row below: every contribution from above is in
            b0 = b1;
            b1 = bn;
            if (lane == 31 && c >= 0) {
                out_slots[c] = make_uint2(out_h, out_e);
                const uint32_t done = (uint32_t)c + 1;
                if (done % p.publish == 0 || done == cols + 1) {
                    cuda::atomic_ref<uint32_t, cuda::thread_scope_device>(p.progress[band]).store(done, cuda::memory_order_release);
                }
            }
        }
        if (below_ok && c + 2 >= 0 && c + 2 < (int64_t)cols) pf = load_rgb(p.img, p.stride, R + 1, (uint32_t)(c + 2));
        // every read of the original row below happens before lane i+1 overwrites it
        __syncwarp();
        hv = __shfl_up_sync(0xffffffffu, out_h, 1);
        ea = __shfl_up_sync(0xffffffffu, out_e, 1);
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------------------

template <typename T> void zero_pad_palette(const uint8_t* palette, uint32_t n, T* out) {
    memset(out, 0, sizeof(T));
    memcpy(out->rgb, palette, (size_t)n * 3);
}

struct ColorCount { uint8_t r, g, b; uint32_t count; };

struct ColorBox {
    ColorCount* colors;
    size_t len;
    uint8_t r_min, r_max, g_min, g_max, b_min, b_max;
    uint32_t population;
    uint32_t volume() const {   // quantize.zig:40-48
        if (r_max < r_min || g_max < g_min || b_max < b_min) return 0;
        return ((uint32_t)r_max - r_min + 1) * ((uint32_t)g_max - g_min + 1) * ((uint32_t)b_max - b_min + 1);
    }
    int largest_dimension() const {   // :50-58
        const int r = r_max >= r_min ? r_max - r_min : 0, g = g_max >= g_min ? g_max - g_min : 0, b = b_max >= b_min ? b_max - b_min : 0;
        if (g >= r && g >= b) return 1;
        if (r >= b) return 0;
        return 2;
    }
};

ColorBox make_box(ColorCount* colors, size_t len) {
    ColorBox b{colors, len, 255, 0, 255, 0, 255, 0, 0};
    for (size_t i = 0; i < len; ++i) {
        const ColorCount& c = colors[i];
        b.r_min = std::min(b.r_min, c.r); b.r_max = std::max(b.r_max, c.r);
        b.g_min = std::min(b.g_min, c.g); b.g_max = std::max(b.g_max, c.g);
        b.b_min = std::min(b.b_min, c.b); b.b_max = std::max(b.b_max, c.b);
        b.population += c.count;
    }
    return b;
}

// std.sort.heap (Zig lib/std/sort.zig, heapContext and siftDown): build the heap with siftDown from n/2 - 1 down to 0, then pop the
// maximum to the end.  siftDown takes the larger child (the right one only when left < right) and stops only when child < cur.
struct DimLess {
    int dim;
    bool operator()(const ColorCount& a, const ColorCount& b) const {
        return dim == 0 ? a.r < b.r : (dim == 1 ? a.g < b.g : a.b < b.b);
    }
};
void sift_down(ColorCount* items, size_t target, size_t n, DimLess less) {
    size_t cur = target;
    for (;;) {
        size_t child = 2 * cur + 1;
        if (!(child < n)) break;
        if (child + 1 < n && less(items[child], items[child + 1])) child = child + 1;
        if (less(items[child], items[cur])) break;
        std::swap(items[child], items[cur]);
        cur = child;
    }
}
void heap_sort(ColorCount* items, size_t n, DimLess less) {
    size_t i = n / 2;
    while (i > 0) {
        --i;
        sift_down(items, i, n, less);
    }
    i = n;
    while (i > 0) {
        --i;
        std::swap(items[0], items[i]);
        sift_down(items, 0, i, less);
    }
}

// quantize.zig:239-411, from the colour list in first-touch order.
int median_cut_boxes(std::vector<ColorCount>& list, uint16_t max_colors, uint8_t* palette, uint32_t cap, uint32_t* n) {
    const size_t palette_size = std::min<size_t>(std::min<size_t>(list.size(), max_colors), cap);
    if (palette_size == 0) return ZB_ERR_NO_PALETTE_COLORS;
    if (list.size() == 1) {
        palette[0] = list[0].r; palette[1] = list[0].g; palette[2] = list[0].b;
        *n = 1;
        return ZB_OK;
    }
    std::vector<ColorBox> boxes;
    boxes.push_back(make_box(list.data(), list.size()));
    while (boxes.size() < palette_size) {
        long largest = -1;
        uint64_t largest_score = 0;
        for (size_t i = 0; i < boxes.size(); ++i) {
            const ColorBox& b = boxes[i];
            if (b.len <= 1) continue;
            if (b.r_max <= b.r_min && b.g_max <= b.g_min && b.b_max <= b.b_min) continue;
            const uint64_t score = (uint64_t)b.volume() * (uint64_t)b.population;
            if (score > largest_score) { largest_score = score; largest = (long)i; }
        }
        if (largest < 0) break;
        const ColorBox split = boxes[largest];
        boxes.erase(boxes.begin() + largest);   // orderedRemove
        heap_sort(split.colors, split.len, DimLess{split.largest_dimension()});
        uint64_t total = 0;
        for (size_t i = 0; i < split.len; ++i) total += split.colors[i].count;
        const uint64_t half = total / 2;
        uint64_t acc = 0;
        size_t cut = 0;
        for (size_t i = 0; i < split.len; ++i) {
            acc += split.colors[i].count;
            if (acc >= half) { cut = std::max<size_t>(1, std::min(i + 1, split.len - 1)); break; }
        }
        const ColorBox b1 = make_box(split.colors, cut), b2 = make_box(split.colors + cut, split.len - cut);
        if (b1.len > 0 && b1.r_max >= b1.r_min) boxes.push_back(b1);
        if (b2.len > 0 && b2.r_max >= b2.r_min) boxes.push_back(b2);
    }
    const size_t actual = std::min<size_t>(boxes.size(), cap);
    for (size_t i = 0; i < actual; ++i) {
        const ColorBox& b = boxes[i];
        uint64_t rs = 0, gs = 0, bs = 0, ws = 0;
        for (size_t k = 0; k < b.len; ++k) {
            const ColorCount& c = b.colors[k];
            rs += (uint64_t)c.r * c.count; gs += (uint64_t)c.g * c.count; bs += (uint64_t)c.b * c.count; ws += c.count;
        }
        uint8_t* o = palette + 3 * i;
        if (ws > 0) { o[0] = (uint8_t)(rs / ws); o[1] = (uint8_t)(gs / ws); o[2] = (uint8_t)(bs / ws); }
        else { o[0] = (uint8_t)((b.r_min + b.r_max) / 2); o[1] = (uint8_t)((b.g_min + b.g_max) / 2); o[2] = (uint8_t)((b.b_min + b.b_max) / 2); }
    }
    *n = (uint32_t)actual;
    return ZB_OK;
}

int check_src(const zb_image* src, int pixfmt) {
    if (!src) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if ((uint64_t)src->rows * src->cols > 0 && !src->data) return ZB_ERR_INVALID_ARGUMENT;
    return ZB_OK;
}

template <int SF> void launch_histogram(const zb_image* src, uint32_t* counts, uint32_t* first, cudaStream_t s) {
    mc_histogram<SF><<<row_grid(div_up(src->cols, kTileThreads), src->rows), kTileThreads, 0, s>>>(src->data, src->stride, src->rows,
                                                                                                  src->cols, counts, first);
}

// Device histogram, host cut.  Arguments are checked by the caller.  Waits for the stream.
int median_cut(const zb_image* src, int pixfmt, uint16_t max_colors, uint8_t* palette, uint32_t cap, uint32_t* n, cudaStream_t s) {
    std::vector<ColorCount> list;
    if ((uint64_t)src->rows * src->cols > 0) {
        DeviceInfo di;
        int rc = device_info(&di);
        if (rc) return rc;
        Scratch sc;
        if ((rc = sc.alloc(2 * kLutSize * sizeof(uint32_t), s))) return rc;
        uint32_t* counts = sc.as<uint32_t>();
        uint32_t* first = counts + kLutSize;
        ZB_CUDA(cudaMemsetAsync(counts, 0, kLutSize * sizeof(uint32_t), s));
        ZB_CUDA(cudaMemsetAsync(first, 0xff, kLutSize * sizeof(uint32_t), s));
        switch (pixfmt) {
            case ZB_PIX_U8: launch_histogram<ZB_PIX_U8>(src, counts, first, s); break;
            case ZB_PIX_F32: launch_histogram<ZB_PIX_F32>(src, counts, first, s); break;
            case ZB_PIX_RGB8: launch_histogram<ZB_PIX_RGB8>(src, counts, first, s); break;
            case ZB_PIX_RGBA8: launch_histogram<ZB_PIX_RGBA8>(src, counts, first, s); break;
            default: launch_histogram<ZB_PIX_RGBAF32>(src, counts, first, s); break;
        }
        ZB_LAUNCHED();
        t_last_kernel = "median_cut_histogram";
        std::vector<uint32_t> host(2 * kLutSize);
        ZB_CUDA(cudaMemcpyAsync(host.data(), counts, host.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        // quantize.zig:220-237: the touched keys in first-touch order
        std::vector<std::pair<uint32_t, uint32_t>> touched;   // (first index, key)
        for (uint32_t k = 0; k < (uint32_t)kLutSize; ++k)
            if (host[k]) touched.emplace_back(host[kLutSize + k], k);
        std::sort(touched.begin(), touched.end());
        list.reserve(touched.size());
        for (const auto& tk : touched) {
            const uint32_t k = tk.second;
            const uint8_t r5 = (k >> 10) & 31, g5 = (k >> 5) & 31, b5 = k & 31;
            list.push_back({(uint8_t)((r5 << 3) | (r5 >> 2)), (uint8_t)((g5 << 3) | (g5 >> 2)), (uint8_t)((b5 << 3) | (b5 >> 2)), host[k]});
        }
    }
    return median_cut_boxes(list, max_colors, palette, cap, n);
}

// quantize.zig:414-473
void fixed_6x7x6(uint8_t* p) {
    int i = 0;
    for (int r = 0; r < 6; ++r)
        for (int g = 0; g < 7; ++g)
            for (int b = 0; b < 6; ++b, i += 3) {
                p[i] = (uint8_t)((r * 255 + 2) / 5);
                p[i + 1] = (uint8_t)((g * 255 + 3) / 6);
                p[i + 2] = (uint8_t)((b * 255 + 2) / 5);
            }
}
void web216(uint8_t* p) {
    int i = 0;
    for (int r = 0; r < 6; ++r)
        for (int g = 0; g < 6; ++g)
            for (int b = 0; b < 6; ++b, i += 3) { p[i] = (uint8_t)(r * 51); p[i + 1] = (uint8_t)(g * 51); p[i + 2] = (uint8_t)(b * 51); }
}
const uint8_t kVga16[16 * 3] = {0, 0, 0, 128, 0, 0, 0, 128, 0, 128, 128, 0, 0, 0, 128, 128, 0, 128, 0, 128, 128, 192, 192, 192,
                                128, 128, 128, 255, 0, 0, 0, 255, 0, 255, 255, 0, 0, 0, 255, 255, 0, 255, 0, 255, 255, 255, 255, 255};

template <int SF> int launch_lookup(const zb_image* src, const uint8_t* lut, zb_image* dst, cudaStream_t s) {
    const dim3 grid = row_grid(div_up(src->cols, (size_t)kTileThreads * kTilePx), div_up(src->rows, kTileRows));
    lookup_kernel<SF><<<grid, kTileThreads, 0, s>>>(src->data, src->stride, (uint8_t*)dst->data, dst->stride, src->rows, src->cols, lut);
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_median_cut(const zb_image* src, int pixfmt, uint16_t max_colors, uint8_t* palette, uint32_t cap, uint32_t* n,
                             zb_stream s) {
    int rc = check_src(src, pixfmt);
    if (rc) return rc;
    if (!palette || !n) return ZB_ERR_INVALID_ARGUMENT;
    if ((uint64_t)src->rows * src->cols >= (1ull << 32)) return ZB_ERR_UNSUPPORTED;   // the reference's counts and population are u32
    return median_cut(src, pixfmt, max_colors, palette, cap, n, (cudaStream_t)s);
}

extern "C" int zb_build_palette(const zb_image* src, int pixfmt, int mode, uint16_t max_colors, uint8_t* palette, uint32_t* n,
                                zb_stream s) {
    if (!palette || !n) return ZB_ERR_INVALID_ARGUMENT;
    switch (mode) {
        case ZB_PALETTE_FIXED_6X7X6: fixed_6x7x6(palette); *n = 252; return ZB_OK;
        case ZB_PALETTE_FIXED_VGA16: memcpy(palette, kVga16, sizeof(kVga16)); *n = 16; return ZB_OK;
        case ZB_PALETTE_FIXED_WEB216: web216(palette); *n = 216; return ZB_OK;
        case ZB_PALETTE_ADAPTIVE: break;
        default: return ZB_ERR_INVALID_ARGUMENT;
    }
    int rc = check_src(src, pixfmt);
    if (rc) return rc;
    // quantize.zig:522-525: any medianCut error falls back to the fixed 6x7x6 palette.  A device failure is reported instead.
    rc = (uint64_t)src->rows * src->cols >= (1ull << 32) ? ZB_ERR_UNSUPPORTED
                                                         : median_cut(src, pixfmt, max_colors, palette, 256, n, (cudaStream_t)s);
    if (rc == ZB_ERR_DEVICE_FAILURE) return rc;
    if (rc) {
        fixed_6x7x6(palette);
        *n = 252;
    }
    return ZB_OK;
}

extern "C" int zb_color_lut(const uint8_t* palette, uint32_t n, uint8_t* lut, zb_stream s) {
    if (!palette || !lut || n == 0 || n > 256) return ZB_ERR_INVALID_ARGUMENT;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    Pal pal;
    zero_pad_palette(palette, n, &pal);
    color_lut_kernel<<<kLutSize / 256, 256, 0, (cudaStream_t)s>>>(pal, n, lut);
    ZB_LAUNCHED();
    t_last_kernel = "color_lut";
    return ZB_OK;
}

extern "C" int zb_palette_lookup(const zb_image* src, int pixfmt, const uint8_t* lut, zb_image* dst_u8, zb_stream s_) {
    int rc = check_src(src, pixfmt);
    if (rc) return rc;
    if (!lut || !dst_u8) return ZB_ERR_INVALID_ARGUMENT;
    if (dst_u8->rows != src->rows || dst_u8->cols != src->cols) return ZB_ERR_DIMENSION_MISMATCH;
    if ((uint64_t)src->rows * src->cols == 0) return ZB_OK;
    if (!dst_u8->data) return ZB_ERR_INVALID_ARGUMENT;
    DeviceInfo di;
    if ((rc = device_info(&di))) return rc;
    cudaStream_t s = (cudaStream_t)s_;
    t_last_kernel = "palette_lookup";
    switch (pixfmt) {
        case ZB_PIX_U8: return launch_lookup<ZB_PIX_U8>(src, lut, dst_u8, s);
        case ZB_PIX_F32: return launch_lookup<ZB_PIX_F32>(src, lut, dst_u8, s);
        case ZB_PIX_RGB8: return launch_lookup<ZB_PIX_RGB8>(src, lut, dst_u8, s);
        case ZB_PIX_RGBA8: return launch_lookup<ZB_PIX_RGBA8>(src, lut, dst_u8, s);
        default: return launch_lookup<ZB_PIX_RGBAF32>(src, lut, dst_u8, s);
    }
}

extern "C" int zb_dither(zb_image* img, int pixfmt, const uint8_t* palette, uint32_t n, const uint8_t* lut, int mode, zb_stream s_) {
    if (!img || !palette || !lut || n == 0 || n > 256) return ZB_ERR_INVALID_ARGUMENT;
    if (mode < ZB_DITHER_NONE || mode > ZB_DITHER_AUTO) return ZB_ERR_INVALID_ARGUMENT;
    if (pixfmt != ZB_PIX_RGB8) return ZB_ERR_UNSUPPORTED;
    if (mode == ZB_DITHER_NONE || mode == ZB_DITHER_AUTO) return ZB_OK;   // dither.zig:36
    const uint32_t rows = img->rows, cols = img->cols;
    if ((uint64_t)rows * cols == 0) return ZB_OK;
    if (!img->data) return ZB_ERR_INVALID_ARGUMENT;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)s_;
    Pal pal;
    zero_pad_palette(palette, n, &pal);
    if (mode == ZB_DITHER_ORDERED) {
        const dim3 grid = row_grid(div_up(cols, (size_t)kTileThreads * kTilePx), div_up(rows, kTileRows));
        ordered_kernel<<<grid, kTileThreads, 0, s>>>((uint8_t*)img->data, img->stride, rows, cols, lut, pal);
        ZB_LAUNCHED();
        t_last_kernel = "dither_ordered";
        return ZB_OK;
    }
    const uint32_t nbands = (rows + 31) / 32;
    const size_t slot_bytes = (size_t)nbands * (cols + 1) * sizeof(uint2);
    const size_t ctr_bytes = ((size_t)nbands + 1) * sizeof(uint32_t);
    Scratch sc;
    if ((rc = sc.alloc(slot_bytes + ctr_bytes, s))) return rc;
    DiffuseParams p;
    p.img = (uint8_t*)img->data;
    p.stride = img->stride;
    p.rows = rows;
    p.cols = cols;
    p.lut = lut;
    p.slots = sc.as<uint2>();
    p.progress = (uint32_t*)((uint8_t*)sc.p + slot_bytes);
    p.ticket = p.progress + nbands;
    p.nbands = nbands;
    p.publish = (uint32_t)g_tune_dither_publish.load();
    ZB_CUDA(cudaMemsetAsync(p.progress, 0, ctr_bytes, s));   // every call starts from zero counters and a zero ticket
    const unsigned grid = div_up(nbands, kDiffuseWarps);
    if (mode == ZB_DITHER_FLOYD_STEINBERG) {
        diffuse_kernel<false><<<grid, 32 * kDiffuseWarps, 0, s>>>(p, pal);
        t_last_kernel = "dither_floyd_steinberg";
    } else {
        diffuse_kernel<true><<<grid, 32 * kDiffuseWarps, 0, s>>>(p, pal);
        t_last_kernel = "dither_atkinson";
    }
    ZB_LAUNCHED();
    return ZB_OK;
}
