// zb_jpeg_common.cuh -- what the baseline JPEG encoder (zb_jpeg.cu) and decoder (zb_jpeg_decode.cu) share: the zigzag order and
// the exclusive scan of u32 items into u64 offsets (per-tile partials, one CTA over the partials, then the tiles again).
// Everything is in an unnamed namespace, so each translation unit gets its own copy of the kernels.
#pragma once
#include <cstdint>

#include "zb_internal.h"

namespace zb {
namespace {

// Zigzag scan order: scan position i reads natural index kZigzag[i] (jpeg.zig:49-58, T.81 Figure A.6).
constexpr uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

constexpr int kThreads = 256;           // every other kernel
constexpr int kScanPer = 8;             // items per thread of the scan
constexpr int kScanTile = kThreads * kScanPer;
constexpr int kPartsThreads = 1024;

// Block-wide exclusive scan of one u64 per thread (kThreads threads); *total receives the block's sum.
__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t* total) {
    __shared__ uint64_t warp_sums[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    uint64_t before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
        if (w < warp) before += warp_sums[w];
        sum += warp_sums[w];
    }
    __syncthreads();   // warp_sums may be reused by the caller's next scan
    *total = sum;
    return before + incl - v;
}

// Stage 3 (and the stuffing counts): exclusive prefix sums of u32 items into u64 offsets, off[n] = the total.
__global__ void __launch_bounds__(kThreads) scan_reduce(const uint32_t* __restrict__ v, uint64_t n, uint64_t* __restrict__ part) {
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile;
    uint64_t s = 0;
#pragma unroll
    for (int i = 0; i < kScanPer; ++i) {
        const uint64_t idx = base + (uint64_t)i * kThreads + threadIdx.x;
        if (idx < n) s += v[idx];
    }
    uint64_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) part[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kPartsThreads) scan_parts(uint64_t* __restrict__ part, uint64_t nparts, uint64_t* __restrict__ total_out) {
    __shared__ uint64_t warp_sums[kPartsThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t carry = 0;
    for (uint64_t base = 0; base < nparts; base += kPartsThreads) {
        const uint64_t idx = base + threadIdx.x;
        const uint64_t v = idx < nparts ? part[idx] : 0;
        uint64_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        uint64_t before = 0, sum = 0;
        for (int w = 0; w < kPartsThreads / 32; ++w) {
            if (w < warp) before += warp_sums[w];
            sum += warp_sums[w];
        }
        if (idx < nparts) part[idx] = carry + before + incl - v;
        carry += sum;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total_out = carry;
}

__global__ void __launch_bounds__(kThreads) scan_down(const uint32_t* __restrict__ v, uint64_t n, const uint64_t* __restrict__ part,
                                                      uint64_t* __restrict__ off) {
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanPer;
    uint32_t x[kScanPer];
    uint64_t s = 0;
#pragma unroll
    for (int i = 0; i < kScanPer; ++i) {
        x[i] = base + i < n ? v[base + i] : 0;
        s += x[i];
    }
    uint64_t total;
    uint64_t run = part[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
    for (int i = 0; i < kScanPer; ++i) {
        if (base + i < n) off[base + i] = run;
        run += x[i];
    }
}

// Exclusive scan of n u32 items into off[0..n], off[n] the total.  part: one u64 per tile.
int scan(const uint32_t* v, uint64_t n, uint64_t* part, uint64_t* off, cudaStream_t s) {
    const uint64_t tiles = (n + kScanTile - 1) / kScanTile;
    scan_reduce<<<(unsigned)tiles, kThreads, 0, s>>>(v, n, part);
    ZB_LAUNCHED();
    scan_parts<<<1, kPartsThreads, 0, s>>>(part, tiles, off + n);
    ZB_LAUNCHED();
    scan_down<<<(unsigned)tiles, kThreads, 0, s>>>(v, n, part, off);
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace
}  // namespace zb
