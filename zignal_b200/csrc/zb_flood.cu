// zb_flood.cu -- Image.floodFill (image.zig:831-840, image/flood_fill.zig:59-131) as connected-component labelling by union-find.
//
// The reference walks an explicit stack from the seed.  Its result does not depend on the visiting order: check() reads a neighbour only
// while it is unvisited, and unvisited pixels are never written, so every comparison sees original values.  The filled set is therefore
//   .seed     : the seed plus every pixel joined to it by a path (4- or 8-connected) whose pixels, the seed excepted, pass
//               dist(p, seed) <= threshold;
//   .neighbor : the seed's component in the graph whose edges join adjacent p, q with dist(p, q) <= threshold (dist is symmetric).
// Both are components of one undirected graph on the pixels, with the edge predicate
//   .seed     : pass(p) && pass(q),  pass(x) = x is the seed || dist(x, seed) <= threshold
//   .neighbor : dist(p, q) <= threshold,
// so a labelling of that graph and a fill of every pixel whose root is the seed's root reproduce the reference bit for bit.
//
// Three launches on the caller's stream, no host round trip (the seed value and the seed's root are read on the device):
//   flood_local  : one 32 x 16 tile per CTA.  Pixel values (.neighbor) or pass bits (.seed) in shared memory; the horizontal runs of
//                  each row come from one warp ballot, then each thread unions its forward edges to the next row inside the tile (down;
//                  down-left and down-right for 8-connectivity) with an atomicMin union-find on shared labels, then writes the global
//                  index r * cols + c of its local root into the u32 label plane (scratch, 4 B / pixel).  A local root is the smallest index of its local component, so labels never exceed their own index.
//   flood_border : one thread per tile-border pixel (last row, first and last column: 62 per tile) unions the forward edges that leave
//                  the tile -- including the diagonals at tile corners -- with the same union-find on the global plane.
//   flood_fill   : per pixel, its root against the seed's root; equal ones get fill_value.  The only kernel that writes the image, after
//                  every read of it has finished, so working in place is race-free; writes honour `stride` and stay inside the view.
//
// Union (Playne & Hawick, IEEE TPDS 2018): roots are linked larger-under-smaller with atomicMin; an atomicMin that finds its target no
// longer a root retries with the value it found, so no link is lost.  find() halves paths with atomicMin as well, which never raises a
// label and only ever points a pixel at one of its ancestors; without it, chains along a maze-like region grow with the number of tiles
// the region crosses.  Nothing iterates to a fixed point: each kernel finishes in one pass for any region shape.
#include <type_traits>

#include "zb_internal.h"

namespace zb {
namespace {

constexpr int kTileW = 32, kTileH = 16;            // flood_local: one pixel per thread
constexpr int kBorderPerTile = 64;                 // flood_border: 62 pixels per tile, 2 idle lanes
constexpr int kBorderTiles = 4;                    // tiles per flood_border CTA
constexpr int kFillThreads = 256;

struct Rgb8 { uint8_t r, g, b; };
struct alignas(4) Rgba8 { uint8_t r, g, b, a; };
struct alignas(16) RgbaF32 { float r, g, b, a; };

__device__ __forceinline__ double sq_add(double sum, double x1, double x2) {
    const double d = __dsub_rn(x1, x2);
    return __dadd_rn(sum, __dmul_rn(d, d));
}

// flood_fill.zig:28-51 pixelDistance, in f64: |a - b| for scalars; for the colour structs sum += d * d over r, g, b (and a), each
// product and sum rounded separately, then a correctly rounded square root.
__device__ __forceinline__ double pixel_distance(uint8_t a, uint8_t b) { return fabs(__dsub_rn((double)a, (double)b)); }
__device__ __forceinline__ double pixel_distance(float a, float b) { return fabs(__dsub_rn((double)a, (double)b)); }
__device__ __forceinline__ double pixel_distance(Rgb8 a, Rgb8 b) {
    double s = 0.0;
    s = sq_add(s, a.r, b.r);
    s = sq_add(s, a.g, b.g);
    s = sq_add(s, a.b, b.b);
    return __dsqrt_rn(s);
}
__device__ __forceinline__ double pixel_distance(Rgba8 a, Rgba8 b) {
    double s = 0.0;
    s = sq_add(s, a.r, b.r);
    s = sq_add(s, a.g, b.g);
    s = sq_add(s, a.b, b.b);
    s = sq_add(s, a.a, b.a);
    return __dsqrt_rn(s);
}
__device__ __forceinline__ double pixel_distance(RgbaF32 a, RgbaF32 b) {
    double s = 0.0;
    s = sq_add(s, a.r, b.r);
    s = sq_add(s, a.g, b.g);
    s = sq_add(s, a.b, b.b);
    s = sq_add(s, a.a, b.a);
    return __dsqrt_rn(s);
}

template <typename T> __device__ __forceinline__ T load_px(const T* img, size_t stride, uint32_t r, uint32_t c) {
    return img[(size_t)r * stride + c];
}

template <typename T> struct Params {
    T* img;
    uint32_t* labels;            // rows x cols, dense
    size_t stride;
    uint32_t rows, cols;
    uint32_t seed_r, seed_c;
    double threshold;
    T fill;
};

// The edge predicate.  `<=` in f64: a NaN distance or threshold is no edge, as in the reference.
template <typename T, bool SEED> struct Edge;
template <typename T> struct Edge<T, true> {   // .seed: pass(p) && pass(q), the seed forced to pass
    T seed;
    double t;
    __device__ __forceinline__ bool pass(const Params<T>& p, uint32_t r, uint32_t c) const {
        return (r == p.seed_r && c == p.seed_c) || pixel_distance(load_px(p.img, p.stride, r, c), seed) <= t;
    }
};
template <typename T> struct Edge<T, false> {  // .neighbor: dist(p, q) <= t
    double t;
    __device__ __forceinline__ bool operator()(T a, T b) const { return pixel_distance(a, b) <= t; }
};

// ---- union-find ---------------------------------------------------------------------------------------------------------------------
// Invariant: labels[x] <= x, and labels[x] lies in x's component; x is a root iff labels[x] == x.

__device__ __forceinline__ uint32_t find_root(uint32_t* L, uint32_t x) {
    for (;;) {
        const uint32_t p = __ldcg(L + x);
        if (p == x) return x;
        const uint32_t g = __ldcg(L + p);
        if (g == p) return p;
        atomicMin(L + x, g);   // path halving: x now points at its grandparent (or lower, if another thread got there first)
        x = g;
    }
}

__device__ __forceinline__ void union_roots(uint32_t* L, uint32_t a, uint32_t b) {
    for (;;) {
        a = find_root(L, a);
        b = find_root(L, b);
        if (a == b) return;
        if (a > b) { const uint32_t t = a; a = b; b = t; }
        const uint32_t old = atomicMin(L + b, a);
        if (old == b) return;   // b was still a root: linked
        b = old;                // b was linked meanwhile (to old); join a with old instead
    }
}

// The same on shared-memory labels inside one tile.
__device__ __forceinline__ int find_local(int* L, int x) {
    volatile int* V = L;
    for (;;) {
        const int p = V[x];
        if (p == x) return x;
        const int g = V[p];
        if (g == p) return p;
        atomicMin(L + x, g);
        x = g;
    }
}
__device__ __forceinline__ void union_local(int* L, int a, int b) {
    for (;;) {
        a = find_local(L, a);
        b = find_local(L, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(L + b, a);
        if (old == b) return;
        b = old;
    }
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------------

template <typename T, bool SEED, bool EIGHT>
__global__ void __launch_bounds__(kTileW * kTileH) flood_local(Params<T> p) {
    __shared__ int lab[kTileH * kTileW];
    __shared__ typename std::conditional<SEED, uint8_t, T>::type key[kTileH][kTileW];   // pass bit (.seed) or pixel value (.neighbor)
    const int tile_r = ZB_GRID_ROW();
    if ((uint32_t)tile_r * kTileH >= p.rows) return;   // uniform per block
    const int tx = threadIdx.x, ty = threadIdx.y, t = ty * kTileW + tx;
    const uint32_t r0 = (uint32_t)tile_r * kTileH, c0 = blockIdx.x * kTileW;
    const uint32_t r = r0 + ty, c = c0 + tx;
    const bool in = r < p.rows && (uint64_t)c0 + tx < p.cols;   // 64-bit: c0 + tx may pass 2^32 in the last tile of a wide image
    const int h = p.rows - r0 < kTileH ? (int)(p.rows - r0) : kTileH;   // this tile's extent
    const int w = p.cols - c0 < kTileW ? (int)(p.cols - c0) : kTileW;
    if (in) {
        if constexpr (SEED) {
            const Edge<T, true> e{load_px(p.img, p.stride, p.seed_r, p.seed_c), p.threshold};
            key[ty][tx] = e.pass(p, r, c);
        } else {
            key[ty][tx] = load_px(p.img, p.stride, r, c);
        }
    }
    __syncthreads();
    auto edge = [&](int y, int x) -> bool {
        if constexpr (SEED) return key[ty][tx] && key[y][x];
        else return Edge<T, false>{p.threshold}(key[ty][tx], key[y][x]);
    };
    // Each warp is one tile row: its horizontal runs come from one ballot, and every pixel starts out pointing at its run's first pixel
    // (lane s starts a run when s == 0 or s - 1 has no edge to s), so only the vertical and diagonal edges need the union-find.
    const unsigned joined = __ballot_sync(0xffffffffu, in && tx + 1 < w && edge(ty, tx + 1));   // bit x: x joined to x + 1
    const unsigned starts = (~joined << 1) | 1u;
    lab[t] = ty * kTileW + 31 - __clz(starts & ((2u << tx) - 1u));
    __syncthreads();
    if (in) {
        if (ty + 1 < h) {
            if (edge(ty + 1, tx)) union_local(lab, t, t + kTileW);
            if constexpr (EIGHT) {
                if (tx > 0 && edge(ty + 1, tx - 1)) union_local(lab, t, t + kTileW - 1);
                if (tx + 1 < w && edge(ty + 1, tx + 1)) union_local(lab, t, t + kTileW + 1);
            }
        }
    }
    __syncthreads();
    if (in) {
        const int root = find_local(lab, t);
        p.labels[(size_t)r * p.cols + c] = (r0 + (uint32_t)(root / kTileW)) * p.cols + c0 + (uint32_t)(root % kTileW);
    }
}

// Forward edges of (r, c) that leave its tile, unioned on the global plane.  Per tile, lanes 0..31 take the last row, 32..46 the last
// column and 48..62 the first column (rows 0..14 of each; row 15 of both columns belongs to the last row).
template <typename T, bool SEED, bool EIGHT>
__global__ void __launch_bounds__(kBorderPerTile * kBorderTiles) flood_border(Params<T> p) {
    const int tile_r = ZB_GRID_ROW();
    const uint32_t r0 = (uint32_t)tile_r * kTileH;
    if (r0 >= p.rows) return;
    const int lane = threadIdx.x % kBorderPerTile;
    const uint64_t c0_wide = ((uint64_t)blockIdx.x * kBorderTiles + threadIdx.x / kBorderPerTile) * kTileW;
    if (c0_wide >= p.cols) return;   // a tile past the image (the last CTA's share)
    const uint32_t c0 = (uint32_t)c0_wide;
    uint32_t r, c;
    if (lane < 32) { r = r0 + kTileH - 1; c = c0 + lane; }
    else if (lane < 47) { r = r0 + (lane - 32); c = c0 + kTileW - 1; }
    else if (lane >= 48 && lane < 63) { r = r0 + (lane - 48); c = c0; }
    else return;
    if (r >= p.rows || (uint64_t)c0 + (c - c0) >= p.cols) return;
    const uint32_t i = r * p.cols + c;
    const bool last_col = c == c0 + kTileW - 1, last_row = r == r0 + kTileH - 1, first_col = c == c0;
    const bool right = c + 1 < p.cols && last_col;   // the right neighbour is in another tile
    const bool down = r + 1 < p.rows;
    if constexpr (SEED) {
        const Edge<T, true> e{load_px(p.img, p.stride, p.seed_r, p.seed_c), p.threshold};
        if (!e.pass(p, r, c)) return;
        if (right && e.pass(p, r, c + 1)) union_roots(p.labels, i, i + 1);
        if (down && last_row) {
            if (e.pass(p, r + 1, c)) union_roots(p.labels, i, i + p.cols);
        }
        if constexpr (EIGHT) {
            if (down && c > 0 && (last_row || first_col) && e.pass(p, r + 1, c - 1)) union_roots(p.labels, i, i + p.cols - 1);
            if (down && c + 1 < p.cols && (last_row || last_col) && e.pass(p, r + 1, c + 1)) union_roots(p.labels, i, i + p.cols + 1);
        }
    } else {
        const Edge<T, false> e{p.threshold};
        const T v = load_px(p.img, p.stride, r, c);
        if (right && e(v, load_px(p.img, p.stride, r, c + 1))) union_roots(p.labels, i, i + 1);
        if (down && last_row && e(v, load_px(p.img, p.stride, r + 1, c))) union_roots(p.labels, i, i + p.cols);
        if constexpr (EIGHT) {
            if (down && c > 0 && (last_row || first_col) && e(v, load_px(p.img, p.stride, r + 1, c - 1))) union_roots(p.labels, i, i + p.cols - 1);
            if (down && c + 1 < p.cols && (last_row || last_col) && e(v, load_px(p.img, p.stride, r + 1, c + 1)))
                union_roots(p.labels, i, i + p.cols + 1);
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kFillThreads) flood_fill(Params<T> p) {
    __shared__ uint32_t seed_root;
    const int r = ZB_GRID_ROW();
    if ((uint32_t)r >= p.rows) return;   // uniform per block
    if (threadIdx.x == 0) seed_root = find_root(p.labels, p.seed_r * p.cols + p.seed_c);
    __syncthreads();
    const uint64_t c_wide = (uint64_t)blockIdx.x * kFillThreads + threadIdx.x;
    if (c_wide >= p.cols) return;
    const uint32_t c = (uint32_t)c_wide;
    const uint32_t i = (uint32_t)r * p.cols + c;
    uint32_t l = p.labels[i];
    if (l != seed_root) l = find_root(p.labels, l);   // most pixels point at their local root, most local roots at the region's root
    if (l == seed_root) {
        p.img[(size_t)r * p.stride + c] = p.fill;
    }
}

template <typename T, bool SEED, bool EIGHT>
int launch(Params<T> p, cudaStream_t s) {
    const size_t tiles_y = div_up(p.rows, kTileH), tiles_x = div_up(p.cols, kTileW);
    flood_local<T, SEED, EIGHT><<<row_grid((unsigned)tiles_x, tiles_y), dim3(kTileW, kTileH), 0, s>>>(p);
    ZB_LAUNCHED();
    flood_border<T, SEED, EIGHT><<<row_grid(div_up(tiles_x, kBorderTiles), tiles_y), kBorderPerTile * kBorderTiles, 0, s>>>(p);
    ZB_LAUNCHED();
    flood_fill<T><<<row_grid(div_up(p.cols, kFillThreads), p.rows), kFillThreads, 0, s>>>(p);
    ZB_LAUNCHED();
    t_last_kernel = "flood_fill";
    return ZB_OK;
}

template <typename T>
int run(const zb_image* img, uint32_t sr, uint32_t sc, const void* fill, double threshold, bool eight, bool seed, cudaStream_t s) {
    Scratch sc_labels;
    int rc = sc_labels.alloc((size_t)img->rows * img->cols * sizeof(uint32_t), s);
    if (rc) return rc;
    Params<T> p;
    p.img = (T*)img->data;
    p.labels = sc_labels.as<uint32_t>();
    p.stride = img->stride;
    p.rows = img->rows;
    p.cols = img->cols;
    p.seed_r = sr;
    p.seed_c = sc;
    p.threshold = threshold;
    memcpy(&p.fill, fill, sizeof(T));
    if (seed) return eight ? launch<T, true, true>(p, s) : launch<T, true, false>(p, s);
    return eight ? launch<T, false, true>(p, s) : launch<T, false, false>(p, s);
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" int zb_flood_fill(zb_image* img, int pixfmt, uint32_t start_row, uint32_t start_col, const void* fill_value, double threshold,
                             int connectivity, int mode, zb_stream s_) {
    if (!img) return ZB_ERR_INVALID_ARGUMENT;
    if (channels_of(pixfmt) == 0) return ZB_ERR_UNSUPPORTED;
    if ((connectivity != 4 && connectivity != 8) || (mode != ZB_FLOOD_SEED && mode != ZB_FLOOD_NEIGHBOR) || !fill_value)
        return ZB_ERR_INVALID_ARGUMENT;
    if (start_row >= img->rows || start_col >= img->cols) return ZB_ERR_OUT_OF_BOUNDS;   // flood_fill.zig:68-70
    if ((uint64_t)img->rows * img->cols >= (1ull << 32)) return ZB_ERR_UNSUPPORTED;       // u32 labels index a dense rows x cols plane
    if (!img->data) return ZB_ERR_INVALID_ARGUMENT;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)s_;
    const bool eight = connectivity == 8, seed = mode == ZB_FLOOD_SEED;
    switch (pixfmt) {
        case ZB_PIX_U8: return run<uint8_t>(img, start_row, start_col, fill_value, threshold, eight, seed, s);
        case ZB_PIX_F32: return run<float>(img, start_row, start_col, fill_value, threshold, eight, seed, s);
        case ZB_PIX_RGB8: return run<Rgb8>(img, start_row, start_col, fill_value, threshold, eight, seed, s);
        case ZB_PIX_RGBA8: return run<Rgba8>(img, start_row, start_col, fill_value, threshold, eight, seed, s);
        case ZB_PIX_RGBAF32: return run<RgbaF32>(img, start_row, start_col, fill_value, threshold, eight, seed, s);
    }
    return ZB_ERR_UNSUPPORTED;
}
