// zb_rotate_tile.cu -- Image.rotateInto for Rgba(u8), bilinear, `.zero` border (BASELINE config 4) from shared-memory source tiles.
// Reference: transforms.zig:189-211 (the inverse-mapped loop; every coordinate is the reference's own unfused f32 sequence),
// interpolation.zig:313-368 (bilinear: out-of-range neighbours are zero pixels under .zero, integer lerp with
// fx = @round(frac * 256) and +32768 rounding).
//
// The gather kernel of zb_warp.cu spends ~130 instructions per interior pixel, most of them on 64-bit addressing, edge tests and
// four scattered global loads.  Here a CTA owns a 64 x 64 destination tile:
//   * the source coordinates are monotone in the column and in the row (every step of the formula is a monotone f32 operation), so
//     the four corners of the tile bound the source footprint exactly; TMA loads that bounding box (<= 95 x 92 pixels for any
//     angle; the start column rounded down to a 16-byte boundary, which TMA insists on) into shared memory as 8-row boxes of a
//     {cols, rows, frames} tensor map.  TMA fills what lies outside the image with
//     zeros, which IS the `.zero` border: no edge test per sample, and a tile whose footprint misses the image is only zero stores;
//   * floor(x) and @round(256 * frac(x)) come out of ONE magic-number add per axis: round-half-up(256 x) = floor(256 x + 1/2)
//     = 256 * floor(x) + fx with fx = 256 carried into the integer part (left + 1 with weight 0 is the same sample as left with
//     weight 256), computed as fma.rm(x, 256, 0.5) (rounding down never crosses an integer) + 1.5 * 2^23 in round-down mode: the
//     low byte of the sum's bit pattern is the weight, the bits above it the tile-relative column.  No conversion instructions;
//   * a warp covers an 8 x 4 pixel patch per step, so its shared-memory footprint is a ~9 x 9 pixel patch for any angle; the tile
//     pitch of 104 words (== 8 mod 32) keeps those four rows in distinct banks; stores are 32-byte row segments.
// The terms of the coordinate that depend on the row only (sin * dy, cos * dy) are tabulated once per tile.
#include <cuda.h>

#include "zb_internal.h"
#include "zb_sample.cuh"
#include "zb_tma.cuh"
#include "zb_warp.h"

namespace zb {

namespace {

constexpr int RT_T = 64;                 // destination tile edge
constexpr int RT_P = 104;                // shared tile pitch in pixels (TMA box width)
constexpr int RT_BOXH = 8;               // rows per TMA box
constexpr int RT_MAXH = 96;              // >= 63 * sqrt(2) + 3, multiple of RT_BOXH
constexpr int RT_THREADS = 256;
constexpr uint32_t RT_SMEM_EXTRA = RT_T * 8 + 16 + 16;   // row terms, footprint bounds, mbarrier
constexpr float RT_MAGIC = 12582912.0f;  // 1.5 * 2^23
constexpr int RT_MAGIC_BITS = 0x4B400000;

// Bit pattern of 1.5 * 2^23 + (256 * floor(x) + @round(256 * (x - floor(x)))) (see the header); exact for |x| < 16384
__device__ __forceinline__ int q8_bits(float x) { return __float_as_int(__fadd_rd(__fmaf_rd(x, 256.0f, 0.5f), RT_MAGIC)); }
__device__ __forceinline__ int q8_coord(float x) { return q8_bits(x) - RT_MAGIC_BITS; }

// interpolation.zig:349-367 on four channels with weights in the carried form (fx, fy in [0, 255]; the other weight is 256 - f).
// The sum of the four products is an exact integer, so the order of the two blends is free: vertical first on two 16-bit lanes
// per register (byte * 256 + 128 <= 65408 never carries), the +128 per lane being the reference's +32768 after the horizontal
// weights (which add up to 256); horizontal as L * gx + R * fx = dp2a([L, R], [gx - 1, fx]) + L -- both weights fit a byte.
__device__ __forceinline__ uint32_t bilerp_rgba8_q(uint32_t tl, uint32_t tr, uint32_t bl, uint32_t br, unsigned fx, unsigned fy) {
    const unsigned gy = 256u - fy;
    const uint32_t l02 = (tl & 0x00FF00FFu) * gy + ((bl & 0x00FF00FFu) * fy + 0x00800080u);
    const uint32_t l13 = __byte_perm(tl, 0, 0x4341) * gy + (__byte_perm(bl, 0, 0x4341) * fy + 0x00800080u);
    const uint32_t r02 = (tr & 0x00FF00FFu) * gy + ((br & 0x00FF00FFu) * fy + 0x00800080u);
    const uint32_t r13 = __byte_perm(tr, 0, 0x4341) * gy + (__byte_perm(br, 0, 0x4341) * fy + 0x00800080u);
    const unsigned w = fx * 255u + 255u;   // bytes: (255 - fx) | fx << 8
    const uint32_t c0 = __dp2a_lo(__byte_perm(l02, r02, 0x5410), w, l02 & 0xFFFFu);
    const uint32_t c2 = __dp2a_lo(__byte_perm(l02, r02, 0x7632), w, l02 >> 16);
    const uint32_t c1 = __dp2a_lo(__byte_perm(l13, r13, 0x5410), w, l13 & 0xFFFFu);
    const uint32_t c3 = __dp2a_lo(__byte_perm(l13, r13, 0x7632), w, l13 >> 16);
    return __byte_perm(__byte_perm(c0, c1, 0x0062), __byte_perm(c2, c3, 0x0062), 0x5410);
}

struct TileParams {
    uint32_t* dst;
    unsigned long long dst_stride, dst_image_pitch;   // pixels
    int dst_rows, dst_cols, src_rows, src_cols;
    float cos_a, sin_a, cx, cy, rcx, rcy;
    uint32_t tile_bytes;                              // shared tile: rows(angle) * RT_P * 4
    int max_boxes;                                    // rows(angle) / RT_BOXH
    unsigned slices;                                  // layered_row_grid: z = frame * slices + slice
};

__global__ void __launch_bounds__(RT_THREADS, 4) rotate_tile_rgba8_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ TileParams p) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t tile = smem_u32(smem_raw);
    float2* rowterm = reinterpret_cast<float2*>(smem_raw + p.tile_bytes);
    int4* bounds = reinterpret_cast<int4*>(smem_raw + p.tile_bytes + RT_T * 8);
    const uint32_t bar = tile + p.tile_bytes + RT_T * 8 + 16;

    const int c0 = blockIdx.x * RT_T, r0 = ZB_LAYER_TILE(p.slices) * RT_T;
    if (r0 >= p.dst_rows) return;   // past the last tile (uniform per block)
    const int frame = (int)ZB_LAYER(p.slices);
    const int c1 = min(c0 + RT_T - 1, p.dst_cols - 1), r1 = min(r0 + RT_T - 1, p.dst_rows - 1);
    if (threadIdx.x < 32) {
        // source footprint of the tile: the coordinates of its four corners (transforms.zig:199-209), one corner per lane (mod 4)
        const float dx = (float)((threadIdx.x & 1u) ? c1 : c0) - p.rcx, dy = (float)((threadIdx.x & 2u) ? r1 : r0) - p.rcy;
        const int x = q8_coord((p.cos_a * dx - p.sin_a * dy) + p.cx) >> 8, y = q8_coord((p.sin_a * dx + p.cos_a * dy) + p.cy) >> 8;
        int min_x = min(x, __shfl_xor_sync(0xffffffffu, x, 1)), max_x = max(x, __shfl_xor_sync(0xffffffffu, x, 1));
        int min_y = min(y, __shfl_xor_sync(0xffffffffu, y, 1)), max_y = max(y, __shfl_xor_sync(0xffffffffu, y, 1));
        min_x = min(min_x, __shfl_xor_sync(0xffffffffu, min_x, 2)); max_x = max(max_x, __shfl_xor_sync(0xffffffffu, max_x, 2));
        min_y = min(min_y, __shfl_xor_sync(0xffffffffu, min_y, 2)); max_y = max(max_y, __shfl_xor_sync(0xffffffffu, max_y, 2));
        if (threadIdx.x == 0) {
            *bounds = make_int4(min_x, max_x, min_y, max_y);
            mbar_init(bar, 1);
            fence_barrier_init();
        }
    }
    if (threadIdx.x < RT_T) {
        const float dy = (float)(r0 + (int)threadIdx.x) - p.rcy;
        rowterm[threadIdx.x] = make_float2(p.sin_a * dy, p.cos_a * dy);
    }
    __syncthreads();
    const int4 b4 = *bounds;
    int min_x = b4.x;
    const int max_x = b4.y, min_y = b4.z, max_y = b4.w;
    const int pc = (int)(threadIdx.x >> 5) * 8 + (int)(threadIdx.x & 7u);   // column of the tile this thread produces
    const int pr = (int)((threadIdx.x >> 3) & 3u);                          // its row within every 4-row step
    const int c = c0 + pc;
    unsigned char* outb = reinterpret_cast<unsigned char*>(p.dst + (size_t)frame * p.dst_image_pitch + (size_t)(r0 + pr) * p.dst_stride + (size_t)c);
    const unsigned long long step_bytes = 16ull * p.dst_stride;
    if (c > c1 || r0 + pr > r1) return;                                                     // (thread 0 never leaves here)
    const int nj = (r1 - r0 - pr) / 4 + 1;                                                  // rows r0 + pr + 4 j <= r1
    if (max_x + 1 < 0 || min_x >= p.src_cols || max_y + 1 < 0 || min_y >= p.src_rows) {   // every neighbour of every sample is outside
        for (int j = 0; j < nj; ++j, outb += step_bytes) *reinterpret_cast<uint32_t*>(outb) = 0u;
        return;
    }
    min_x &= ~3;                                                       // TMA: the box must start on a 16-byte boundary (<= 95 columns are used)
    if (threadIdx.x == 0) {
        const int n_boxes = min((max_y - min_y + 2 + RT_BOXH - 1) / RT_BOXH, p.max_boxes);   // rows min_y .. max_y + 1 (the host sized the tile for them)
        mbar_arrive_expect_tx(bar, (uint32_t)n_boxes * RT_BOXH * RT_P * 4);
        for (int b = 0; b < n_boxes; ++b) tma_load_3d(tile + (uint32_t)b * RT_BOXH * RT_P * 4, &tmap, min_x, min_y + b * RT_BOXH, frame, bar);
    }
    const float dx = (float)c - p.rcx;
    const float cos_dx = p.cos_a * dx, sin_dx = p.sin_a * dx;
    // bits = MAGIC_BITS + (column << 8 | weight): the weight is the low byte as it stands; shifts and masks commute with subtracting
    // a multiple of 256, so the tile origin and the shared address of the tile fold into ONE constant added to the address
    const uint32_t a0 = tile - (uint32_t)(((RT_MAGIC_BITS >> 8) + min_y) * (RT_P * 4)) - (uint32_t)(((RT_MAGIC_BITS >> 8) + min_x) * 4);
    while (!mbar_try_wait(bar, 0)) {}
    if (min_x >= 0 && max_x + 1 < p.src_cols && min_y >= 0 && max_y + 1 < p.src_rows) {   // footprint inside the image
#pragma unroll 4
        for (int j = 0; j < nj; ++j) {
            const float2 rt = rowterm[4 * j + pr];
            const float src_x = (cos_dx - rt.x) + p.cx;
            const float src_y = (sin_dx + rt.y) + p.cy;
            const unsigned mx = (unsigned)q8_bits(src_x), my = (unsigned)q8_bits(src_y);
            const uint32_t a = a0 + (my >> 8) * (RT_P * 4) + ((mx >> 6) & ~3u);
            *reinterpret_cast<uint32_t*>(outb) =
                bilerp_rgba8_q(lds32(a), lds32(a + 4), lds32(a + RT_P * 4), lds32(a + RT_P * 4 + 4), mx & 255u, my & 255u);
            outb += step_bytes;
        }
    } else {
        // A tile on the outline of the rotated frame: about two thirds of its pixels lie outside.  An 8 x 4 patch whose samples ALL
        // have their four neighbours outside the image (column + 1 or row + 1 not in [0, size]) is zero without the blend.
        const unsigned kx4 = (unsigned)(((RT_MAGIC_BITS >> 8) - 1) * 4), ky = (unsigned)((RT_MAGIC_BITS >> 8) - 1);
        const unsigned cols4 = (unsigned)p.src_cols * 4u, rows_u = (unsigned)p.src_rows;
#pragma unroll 2
        for (int j = 0; j < nj; ++j) {
            const float2 rt = rowterm[4 * j + pr];
            const float src_x = (cos_dx - rt.x) + p.cx;
            const float src_y = (sin_dx + rt.y) + p.cy;
            const unsigned mx = (unsigned)q8_bits(src_x), my = (unsigned)q8_bits(src_y);
            const unsigned x4 = (mx >> 6) & ~3u, yy = my >> 8;
            const bool outside = (x4 - kx4) > cols4 || (yy - ky) > rows_u;
            uint32_t v = 0u;
            if (!__all_sync(__activemask(), outside)) {
                const uint32_t a = a0 + yy * (RT_P * 4) + x4;
                v = bilerp_rgba8_q(lds32(a), lds32(a + 4), lds32(a + RT_P * 4), lds32(a + RT_P * 4 + 4), mx & 255u, my & 255u);
            }
            *reinterpret_cast<uint32_t*>(outb) = v;
            outb += step_bytes;
        }
    }
}

}  // namespace

// Returns ZB_ERR_UNSUPPORTED when the tile kernel does not apply (the caller then takes the gather kernel).
int rotate_tile_rgba8(const zb_image* src, unsigned long long spitch, zb_image* dst, unsigned long long dpitch, uint32_t n, const RotParams& rp,
                      cudaStream_t s) {
    if (rp.method != ZB_INTERP_BILINEAR || rp.border != ZB_BORDER_ZERO) return ZB_ERR_UNSUPPORTED;
    // zb_rotate_into_cs takes cos / sin from the caller: the footprint bound below needs an actual rotation
    if (!(std::fabs((double)rp.cos_a) + std::fabs((double)rp.sin_a) <= 1.4143)) return ZB_ERR_UNSUPPORTED;
    if (src->rows == 0 || src->cols == 0 || src->rows > 8192 || src->cols > 8192 || dst->rows > 16384 || dst->cols > 16384) return ZB_ERR_UNSUPPORTED;
    if (n > 65535 || ((uintptr_t)src->data & 15) || (src->stride & 3) || (n > 1 && (spitch & 3)) || ((uintptr_t)dst->data & 3)) return ZB_ERR_UNSUPPORTED;
    EncodeTiledFn encode = encode_tiled_fn();
    if (!encode) return ZB_ERR_UNSUPPORTED;
    CUtensorMap tmap;
    const cuuint64_t gdim[3] = {(cuuint64_t)src->cols, (cuuint64_t)src->rows, (cuuint64_t)n};
    const cuuint64_t frame_bytes = n > 1 ? (cuuint64_t)spitch * 4 : (cuuint64_t)src->rows * src->stride * 4;
    const cuuint64_t gstr[2] = {(cuuint64_t)src->stride * 4, frame_bytes};
    const cuuint32_t box[3] = {(cuuint32_t)RT_P, (cuuint32_t)RT_BOXH, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    if (encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, src->data, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return ZB_ERR_UNSUPPORTED;
    TileParams p;
    p.dst = (uint32_t*)dst->data;
    p.dst_stride = dst->stride;
    p.dst_image_pitch = dpitch;
    p.dst_rows = (int)dst->rows; p.dst_cols = (int)dst->cols;
    p.src_rows = (int)src->rows; p.src_cols = (int)src->cols;
    p.cos_a = rp.cos_a; p.sin_a = rp.sin_a; p.cx = rp.cx; p.cy = rp.cy; p.rcx = rp.rcx; p.rcy = rp.rcy;
    // rows of the footprint for this angle: (T - 1)(|cos| + |sin|) + 3 (floor spread + the bottom neighbour + slack for the
    // rounding of the coordinate sums), in whole boxes; fewer rows = more resident CTAs to hide the tile load behind
    const double span = (RT_T - 1) * (std::fabs((double)rp.cos_a) + std::fabs((double)rp.sin_a));
    int rows = ((int)std::ceil(span) + 3 + RT_BOXH - 1) / RT_BOXH * RT_BOXH;
    if (rows > RT_MAXH) rows = RT_MAXH;      // (|cos| + |sin| > sqrt 2 only for cos / sin pairs that are not a rotation: the kernel clips)
    p.tile_bytes = (uint32_t)rows * RT_P * 4;
    p.max_boxes = rows / RT_BOXH;
    // (A persistent variant with two tile buffers and TMA prefetch of the next tile was measured slower: 1.11 ms against 0.94 ms
    // for 128 frames -- the per-tile bookkeeping of 512 threads costs more issue slots than the hidden load latency returns.)
    const uint32_t smem = p.tile_bytes + RT_SMEM_EXTRA;   // < 48 KB: no size attribute needed
    // five 40 KB tiles per SM need the largest shared-memory carveout (a per-device hint; setting it is cheap)
    cudaFuncSetAttribute(rotate_tile_rgba8_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    dim3 grid;
    if (layered_row_grid(div_up(dst->cols, RT_T), div_up(dst->rows, RT_T), n, &grid, &p.slices)) return ZB_ERR_UNSUPPORTED;
    rotate_tile_rgba8_kernel<<<grid, RT_THREADS, smem, s>>>(tmap, p);
    t_last_kernel = "rotate_tile_rgba8";
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace zb
