// zb_hough.cu -- HoughTransform (image/hough.zig:10-257): line detection on a binary edge map.
//
// compute (hough.zig:75-139), two launches, no host round trip:
//   hough_compact : one pass over box ∩ image.  Every non-zero pixel becomes one u32 entry of a scratch list, (x_val, y_val) as two i16
//                   halves (|x_val|, |y_val| <= size - 1 <= 32767).  Per-CTA count, one global atomic per CTA; the list order is
//                   arbitrary, which is harmless because the votes are integer counts.
//   hough_vote    : CTA (slice, chunk) owns the T angle columns [slice T, slice T + T) and the chunk-th share of the edge list.  It
//                   keeps size x T u32 counters in shared memory (row rr, column a at rr * T + a), streams its share of the list from
//                   L2 and, per angle, forms rr with the reference's i32 expression.  Thread tid works on angle a = tid % T, so
//                   cos[t] / sin[t] live in registers, and walks its own contiguous part of the share (edge lane tid / T): lanes of one
//                   warp on the same angle hold pixels far apart in the list, which rarely meet on one counter (the atomic serialises
//                   them when they do).  No global atomic is in the vote loop.  The slice is then added into the caller's accumulator:
//                   plainly when the list is not split (the CTA owns those cells), with atomicAdd when several chunks share the columns;
//                   zero counters are skipped.
//                   CTA shape (DESIGN.md section 4): 1024 threads and T = min(8, what fits), measured on an H100 against 256 / 512 threads
//                   and 4 / 16 / 32 columns.  The kernel is bound by the latency of the shared-memory atomics, so resident threads
//                   count most: 8 columns of a 4096 box are 128 KB (one 1024-thread CTA per SM), of a 2048 box 64 KB (two).
// findLines (hough.zig:142-204):
//   hough_peaks   : one thread per interior cell: votes >= threshold and no 8-neighbour strictly greater.  Candidates (score, row, col)
//                   are appended to device scratch (warp-aggregated atomic); only their count and the candidates cross PCIe.
//   host          : sort by (score desc, row asc, col asc) -- std.mem.sort is stable over the row-major scan -- then the greedy NMS and
//                   getLineProperties / createLine / clipLine (:207-257) in f32 (this file's host code is built with -ffp-contract=off;
//                   cosf / sinf are the host libm's, as for rotate's cos and sin).
//
// i32 range (why size <= 32768): |cos[t]| + |sin[t]| <= 65536 (|cos| + |sin| <= sqrt(2), then the / sqrt(2) and the truncation) and
// |x_val|, |y_val| <= size - 1, so |rho| <= 65536 (size - 1) <= 2,147,418,112 < 2^31 for size <= 32768.  offset = 16384 even_size <= 2^29,
// so (rho >> 1) + (offset << 1) <= 1,073,709,056 + 2^30 = 2,147,450,880 < 2^31 as well.  At size 32769 |rho| can reach 2^31 and the
// reference's i32 arithmetic overflows; such sizes return ZB_ERR_UNSUPPORTED.
#include <algorithm>
#include <cmath>
#include <mutex>
#include <vector>

#include "zb_internal.h"

struct zb_hough {
    uint32_t size, even_size;
    std::vector<int32_t> tables;      // cos_table then sin_table (host), 2 * size entries
    mutable std::mutex mu;
    mutable int32_t* d_tables = nullptr;   // device copy, uploaded by the first compute
    mutable bool tables_ready = false;     // the upload into d_tables has completed
};

namespace zb {

std::atomic<int> g_tune_hough_threads{1024};
std::atomic<int> g_tune_hough_max_cols{8};

namespace {

constexpr uint32_t kMaxSize = 32768;
constexpr int kCompactThreads = 256;
constexpr int kCompactPerThread = 4;
constexpr int kCompactSpan = kCompactThreads * kCompactPerThread;   // pixels of one area row per CTA

__device__ __forceinline__ uint32_t pack_xy(int x, int y) { return (uint32_t)(uint16_t)x | ((uint32_t)(uint16_t)y << 16); }

// Block-wide exclusive prefix of `v`; returns the prefix and writes the block total to *total.  All threads must call it.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nwarps ? warp_sums[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += u;
        }
        if (lane < nwarps) warp_sums[lane] = w;   // inclusive warp prefix
    }
    __syncthreads();
    *total = warp_sums[nwarps - 1];
    return incl - v + (warp ? warp_sums[warp - 1] : 0u);
}

// hough.zig:91-105: the non-zero pixels of `area` (w x h at edges) as packed (x_val, y_val).  The area starts at the box's top-left
// corner (the image's starts at 0, 0), so x_val = 2 c - (size - 1) for area column c, and likewise for y.
__global__ void __launch_bounds__(kCompactThreads) hough_compact(const uint8_t* __restrict__ edges, size_t stride, int w, int h, int size_m1,
                                                                  uint32_t* __restrict__ list, uint32_t* __restrict__ count) {
    __shared__ uint32_t warp_sums[kCompactThreads / 32];
    __shared__ uint32_t base;
    const int row = ZB_GRID_ROW();
    if (row >= h) return;   // uniform per block
    const uint8_t* src = edges + (size_t)row * stride;
    const int c0 = blockIdx.x * kCompactSpan + threadIdx.x;
    const int y_val = 2 * row - size_m1;
    uint32_t mask = 0, n = 0;
#pragma unroll
    for (int k = 0; k < kCompactPerThread; ++k) {
        const int c = c0 + k * kCompactThreads;
        if (c < w && src[c] != 0) mask |= 1u << k;
    }
    n = __popc(mask);
    uint32_t total;
    const uint32_t off = block_exclusive_scan(n, warp_sums, &total);
    if (total == 0) return;   // uniform per block
    if (threadIdx.x == 0) base = atomicAdd(count, total);
    __syncthreads();
    uint32_t j = base + off;
#pragma unroll
    for (int k = 0; k < kCompactPerThread; ++k)
        if (mask & (1u << k)) list[j++] = pack_xy(2 * (c0 + k * kCompactThreads) - size_m1, y_val);
}

struct VoteParams {
    const uint32_t* list;
    const uint32_t* count;
    const int32_t* cos_t;   // device tables, size entries each
    const int32_t* sin_t;
    uint32_t* acc;
    size_t acc_stride;
    int size, cols;         // cols = T, angle columns per CTA
    int offset2;            // offset << 1 = 2 * round(65536 even_size / 4)
};

__global__ void __launch_bounds__(1024) hough_vote(VoteParams p) {
    extern __shared__ uint32_t cnt[];   // size x T, row rr at rr * T
    const int T = p.cols;
    const int a = threadIdx.x % T, e = threadIdx.x / T, E = blockDim.x / T;
    const int t = blockIdx.x * T + a;
    const bool active = e < E && t < p.size;
    const size_t cells = (size_t)p.size * T;
    const uint32_t n = *p.count;
    const uint32_t beg = (uint32_t)((uint64_t)n * blockIdx.y / gridDim.y), end = (uint32_t)((uint64_t)n * (blockIdx.y + 1) / gridDim.y);
    if (beg == end) return;   // uniform per block: nothing to add
    for (size_t i = threadIdx.x; i < cells; i += blockDim.x) cnt[i] = 0u;
    __syncthreads();
    if (active) {
        const int c = p.cos_t[t], s = p.sin_t[t];
        const unsigned size = (unsigned)p.size;
        auto vote = [&](uint32_t v) {
            const int x = (int)(int16_t)(v & 0xffffu), y = (int)v >> 16;
            const int rho = x * c + y * s;                     // hough.zig:110, i32 (no overflow for size <= 32768, see the header)
            const int rr = ((rho >> 1) + p.offset2) >> 16;     // :111, arithmetic shifts
            if ((unsigned)rr < size) atomicAdd(&cnt[rr * T + a], 1u);   // :112, 0 <= rr < size
        };
        // each edge lane walks its own contiguous part of the share: neighbouring pixels (neighbours in the list too) would often
        // meet on one counter, pixels far apart in the list rarely do
        uint32_t i = beg + (uint32_t)((uint64_t)(end - beg) * e / E);
        const uint32_t stop = beg + (uint32_t)((uint64_t)(end - beg) * (e + 1) / E);
        for (; i + 3u < stop; i += 4u) {
            const uint32_t v0 = __ldg(p.list + i), v1 = __ldg(p.list + i + 1), v2 = __ldg(p.list + i + 2), v3 = __ldg(p.list + i + 3);
            vote(v0);
            vote(v1);
            vote(v2);
            vote(v3);
        }
        for (; i < stop; ++i) vote(__ldg(p.list + i));
    }
    __syncthreads();
    if (!active) return;
    const bool owned = gridDim.y == 1;
    for (int rr = e; rr < p.size; rr += E) {
        const uint32_t v = cnt[rr * T + a];
        if (!v) continue;
        uint32_t* dst = p.acc + (size_t)rr * p.acc_stride + t;
        if (owned) *dst += v;
        else atomicAdd(dst, v);
    }
}

struct Candidate { uint32_t score, row, col; };

// hough.zig:156-177: interior cells with votes >= threshold and no strictly greater 8-neighbour.
__global__ void hough_peaks(const uint32_t* __restrict__ acc, size_t stride, int rows, int cols, uint32_t threshold,
                            Candidate* __restrict__ out, uint32_t cap, uint32_t* __restrict__ count) {
    const int r = ZB_GRID_ROW() + 1;
    if (r >= rows - 1) return;
    const int c = blockIdx.x * blockDim.x + threadIdx.x + 1;
    bool keep = false;
    uint32_t v = 0;
    if (c < cols - 1) {
        const uint32_t* p = acc + (size_t)r * stride + c;
        v = p[0];
        if (v >= threshold) {
            keep = true;
            for (int dr = -1; dr <= 1 && keep; ++dr)
                for (int dc = -1; dc <= 1; ++dc)
                    if ((dr || dc) && p[(ptrdiff_t)dr * (ptrdiff_t)stride + dc] > v) { keep = false; break; }
        }
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (!m) return;
    const int lane = threadIdx.x & 31;
    uint32_t base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(count, (uint32_t)__popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (keep) {
        const uint32_t idx = base + __popc(m & ((1u << lane) - 1u));
        if (idx < cap) out[idx] = Candidate{v, (uint32_t)r, (uint32_t)c};
    }
}

// ---- host: the f32 line geometry of hough.zig:207-257 ------------------------------------------------------------------------------
struct Line { float angle, radius; uint32_t score; float p1x, p1y, p2x, p2y; };

// :232-257 clipLine (Liang-Barsky) against [0, size] x [0, size]
void clip_line(float rl, float rt, float rr, float rb, float* p1x, float* p1y, float* p2x, float* p2y) {
    float t0 = 0.0f, t1 = 1.0f;
    const float dx = *p2x - *p1x, dy = *p2y - *p1y;
    const float p[4] = {-dx, dx, -dy, dy};
    const float q[4] = {*p1x - rl, rr - *p1x, *p1y - rt, rb - *p1y};
    for (int i = 0; i < 4; ++i) {
        if (p[i] == 0) {
            if (q[i] < 0) return;
        } else {
            const float r = q[i] / p[i];
            if (p[i] < 0) {
                if (r > t1) return;
                if (r > t0) t0 = r;
            } else {
                if (r < t0) return;
                if (r < t1) t1 = r;
            }
        }
    }
    if (t0 > t1) return;
    const float ox = *p1x, oy = *p1y;
    *p1x = ox + t0 * dx;
    *p1y = oy + t0 * dy;
    *p2x = ox + t1 * dx;
    *p2y = oy + t1 * dy;
}

// :214-229 createLine
Line create_line(uint32_t size, float angle, float radius, uint32_t score) {
    const float center = (float)(size - 1) / 2.0f;
    const float theta = (angle + 90.0f) * (float)M_PI / 180.0f;
    const float cos_t = cosf(theta), sin_t = sinf(theta);
    const float pcx = radius * cos_t, pcy = radius * sin_t;
    const float dirx = -sin_t, diry = cos_t;
    const float huge = (float)size * 2.0f;
    Line l;
    l.angle = angle;
    l.radius = radius;
    l.score = score;
    l.p1x = center + pcx + dirx * huge;
    l.p1y = center + pcy + diry * huge;
    l.p2x = center + pcx - dirx * huge;
    l.p2y = center + pcy - diry * huge;
    clip_line(0.0f, 0.0f, (float)size, (float)size, &l.p1x, &l.p1y, &l.p2x, &l.p2y);
    return l;
}

}  // namespace
}  // namespace zb

using namespace zb;

extern "C" {

int zb_hough_create(uint32_t size, const int32_t* cos_table, const int32_t* sin_table, zb_hough** out) {
    if (!out) return ZB_ERR_INVALID_ARGUMENT;
    if (size <= 1) return ZB_ERR_INVALID_ARGUMENT;   // hough.zig:39
    if (size > kMaxSize) return ZB_ERR_UNSUPPORTED;  // i32 range, see the top of this file
    if (!cos_table != !sin_table) return ZB_ERR_INVALID_ARGUMENT;
    zb_hough* h = new zb_hough();
    h->size = size;
    h->even_size = size % 2 == 0 ? size : size - 1;   // :40
    h->tables.resize(2 * (size_t)size);
    if (cos_table) {
        std::copy(cos_table, cos_table + size, h->tables.begin());
        std::copy(sin_table, sin_table + size, h->tables.begin() + size);
    } else {   // :49-56, f64
        const double scale = 65536.0, sqrt_2 = std::sqrt(2.0);
        for (uint32_t t = 0; t < size; ++t) {
            const double theta = (double)t * M_PI / (double)h->even_size;
            h->tables[t] = (int32_t)std::trunc(scale * std::cos(theta) / sqrt_2);
            h->tables[size + t] = (int32_t)std::trunc(scale * std::sin(theta) / sqrt_2);
        }
    }
    *out = h;
    return ZB_OK;
}

int zb_hough_destroy(zb_hough* h) {
    if (h && h->d_tables) cudaFree(h->d_tables);
    delete h;
    return ZB_OK;
}

int zb_hough_compute(const zb_hough* h, const zb_image* edges, uint32_t l, uint32_t t, uint32_t r, uint32_t b, zb_image* acc, zb_stream s_) {
    if (!h || !edges || !acc) return ZB_ERR_INVALID_ARGUMENT;
    const uint32_t box_w = l >= r ? 0 : r - l, box_h = t >= b ? 0 : b - t;   // Rectangle.width / height
    if (box_w != h->size || box_h != h->size) return ZB_ERR_DIMENSION_MISMATCH;   // hough.zig:76
    if (acc->rows != h->size || acc->cols != h->size) return ZB_ERR_DIMENSION_MISMATCH;   // :77
    if (!edges->data && edges->rows && edges->cols) return ZB_ERR_INVALID_ARGUMENT;
    if (!acc->data) return ZB_ERR_INVALID_ARGUMENT;
    // :79 area = box ∩ edges.getRectangle()
    const uint32_t al = l, at = t, ar = std::min(r, edges->cols), ab = std::min(b, edges->rows);
    if (al >= ar || at >= ab) return ZB_OK;
    cudaStream_t s = (cudaStream_t)s_;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    {
        std::lock_guard<std::mutex> lk(h->mu);
        if (!h->tables_ready) {
            // uploaded on the caller's stream, which is synchronised before the tables count as ready: a later compute may run on
            // another stream.  (A plain cudaMemcpy from pageable memory would wait for the legacy NULL stream, and may return
            // before the copy lands.)
            if (!h->d_tables) ZB_CUDA(cudaMalloc(&h->d_tables, h->tables.size() * sizeof(int32_t)));
            ZB_CUDA(cudaMemcpyAsync(h->d_tables, h->tables.data(), h->tables.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
            ZB_CUDA(cudaStreamSynchronize(s));
            h->tables_ready = true;
        }
    }
    const int w = (int)(ar - al), ht = (int)(ab - at);
    const size_t area = (size_t)w * ht;
    Scratch sc;
    if ((rc = sc.alloc((area + 1) * sizeof(uint32_t), s))) return rc;   // the count, then one entry per area pixel
    uint32_t* count = sc.as<uint32_t>();
    uint32_t* list = count + 1;
    ZB_CUDA(cudaMemsetAsync(count, 0, sizeof(uint32_t), s));
    const int size = (int)h->size;
    hough_compact<<<row_grid(div_up(w, kCompactSpan), ht), kCompactThreads, 0, s>>>(
        (const uint8_t*)edges->data + (size_t)at * edges->stride + al, edges->stride, w, ht, size - 1, list, count);
    ZB_LAUNCHED();

    // vote: T columns per CTA from the opt-in shared memory (T >= 1 always: 4 * 32768 B = 128 KB), threads a multiple of T
    const int threads = g_tune_hough_threads.load();
    const size_t smem_cap = di.smem_optin;
    int T = (int)std::min<size_t>(smem_cap / (4 * (size_t)size), (size_t)g_tune_hough_max_cols.load());
    T = std::max(1, std::min({T, size, threads}));
    const size_t smem = (size_t)size * T * sizeof(uint32_t);
    ZB_CUDA(cudaFuncSetAttribute(hough_vote, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    ZB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hough_vote, threads, smem));
    per_sm = std::max(per_sm, 1);
    const size_t slices = div_up(size, T);
    // Split the list when the slices alone do not fill one wave; a chunk keeps at least max(1024, size) pixels of the area (the
    // edge count is only known on the device) so that clearing and flushing the slice stays small next to its votes.
    const size_t wave = (size_t)per_sm * di.sm_count;
    const size_t min_chunk = std::max<size_t>(1024, size);
    size_t chunks = std::max<size_t>(1, std::min((wave + slices - 1) / slices, area / min_chunk));
    chunks = std::min<size_t>(chunks, 65535);
    VoteParams p;
    p.list = list;
    p.count = count;
    p.cos_t = h->d_tables;
    p.sin_t = h->d_tables + size;
    p.acc = (uint32_t*)acc->data;
    p.acc_stride = acc->stride;
    p.size = size;
    p.cols = T;
    p.offset2 = 2 * (int)std::lround(65536.0 * (double)h->even_size / 4.0);   // :84 (an exact integer: 16384 even_size)
    hough_vote<<<dim3((unsigned)slices, (unsigned)chunks), threads, smem, s>>>(p);
    ZB_LAUNCHED();
    t_last_kernel = "hough_vote";
    return ZB_OK;
}

int zb_hough_find_lines(const zb_hough* h, const zb_image* acc, uint32_t threshold, float angle_nms, float radius_nms, zb_hough_line* out,
                        uint32_t cap, uint32_t* n_out, zb_stream s_) {
    if (!h || !acc || !n_out || (cap && !out)) return ZB_ERR_INVALID_ARGUMENT;
    *n_out = 0;
    if (acc->rows < 3 || acc->cols < 3) return ZB_OK;   // hough.zig:154
    if (!acc->data) return ZB_ERR_INVALID_ARGUMENT;
    cudaStream_t s = (cudaStream_t)s_;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const size_t interior = (size_t)(acc->rows - 2) * (acc->cols - 2);
    std::vector<Candidate> cand;
    uint32_t cap_c = (uint32_t)std::min<size_t>(interior, 1u << 18);
    for (;;) {
        Scratch sc;
        if ((rc = sc.alloc(16 + (size_t)cap_c * sizeof(Candidate), s))) return rc;
        uint32_t* count = sc.as<uint32_t>();
        Candidate* buf = (Candidate*)(sc.as<char>() + 16);
        ZB_CUDA(cudaMemsetAsync(count, 0, sizeof(uint32_t), s));
        hough_peaks<<<row_grid(div_up(acc->cols - 2, 256), acc->rows - 2), 256, 0, s>>>((const uint32_t*)acc->data, acc->stride, (int)acc->rows,
                                                                                        (int)acc->cols, threshold, buf, cap_c, count);
        ZB_LAUNCHED();
        uint32_t n = 0;
        ZB_CUDA(cudaMemcpyAsync(&n, count, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        if (n > cap_c) { cap_c = n; continue; }   // more candidates than the first buffer held: once more with room for all
        cand.resize(n);
        if (n) ZB_CUDA(cudaMemcpyAsync(cand.data(), buf, (size_t)n * sizeof(Candidate), cudaMemcpyDeviceToHost, s));
        ZB_CUDA(cudaStreamSynchronize(s));
        break;
    }
    // :179-183 stable sort by score over the row-major scan order
    std::sort(cand.begin(), cand.end(), [](const Candidate& x, const Candidate& y) {
        if (x.score != y.score) return x.score > y.score;
        if (x.row != y.row) return x.row < y.row;
        return x.col < y.col;
    });
    // :185-201 greedy NMS; :207-212 getLineProperties
    const float center = (float)(h->size - 1) / 2.0f, even = (float)h->even_size, sqrt2 = sqrtf(2.0f);
    std::vector<std::pair<float, float>> kept;   // (angle, radius)
    uint32_t n = 0;
    for (const Candidate& c : cand) {
        const float angle = 180.0f * ((float)c.col - center) / even;
        const float radius = ((float)c.row - center) * sqrt2;
        bool too_close = false;
        for (const auto& k : kept) {
            const float da = fabsf(k.first - angle), dr = fabsf(k.second - radius);
            if ((da < angle_nms && dr < radius_nms) || ((180.0f - da) < angle_nms && fabsf(k.second + radius) < radius_nms)) {
                too_close = true;
                break;
            }
        }
        if (too_close) continue;
        kept.emplace_back(angle, radius);
        if (n < cap) {
            const Line l = create_line(h->size, angle, radius, c.score);
            out[n] = zb_hough_line{l.angle, l.radius, l.score, l.p1x, l.p1y, l.p2x, l.p2y};
        }
        ++n;
    }
    *n_out = n;
    return ZB_OK;
}

}  // extern "C"
