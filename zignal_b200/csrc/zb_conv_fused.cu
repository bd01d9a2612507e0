// zb_conv_fused.cu -- single-pass separable convolution of interleaved RGBA f32 for sm_90a.
//
// Replaces convolveSeparablePlane(f32) (reference convolution.zig:441-647) applied per channel.  The
// reference streams the image three times (src -> temp -> dst, with a full temp plane in DRAM); this
// kernel reads every input pixel once and writes every output pixel once:
//
//   * work unit = (row segment) x (strip of TW=256 pixels); units are ordered segment-major so that
//     the CTAs resident at one time cover neighbouring strips of the same segment (their x-halos are
//     then L2 hits, not DRAM reads).  plan_units() gives each CTA one long segment where the grid
//     allows, shorter ones on the edge strips; the sharded kernel keeps bands of ~conv.band_rows rows;
//   * a persistent CTA (one per SM, 256 threads) walks its units in chunks of 8 rows:
//       TMA (cp.async.bulk.tensor.3d, SWIZZLE_128B, zero OOB fill) lands chunk i+2 in a 2-stage ring
//       while the SM runs   H(i): stage -> 24-row shared ring of horizontally filtered rows
//       and                 V(i-2): ring -> registers -> 128-bit coalesced global stores;
//   * both passes are register-blocked 8 outputs per thread along the filter axis (a thread loads
//     8+2*HALF float4 and issues 8*K float4 FMAs), which keeps shared-memory traffic (~120 B/px) and
//     FP32 issue (120 FFMA/px) both under the HBM time per pixel;
//   * shared-memory accesses are conflict-free: the TMA box is {8 px, 34 groups, 8 rows} with the
//     128-byte hardware swizzle keyed on (row*34+group)&7 and a quarter-warp reads 8 consecutive
//     groups; the ring is XOR-swizzled on (x>>3)&7 by hand;
//   * taps are kernel parameters (constant bank operands of the FFMAs), zero-padded to 2*HALF+1.
//
// Arithmetic: acc = 0; acc += px*k, taps ascending, horizontal pass first and its result rounded to
// f32 before the vertical pass -- the reference's order.  EXACT=true keeps mul and add unfused
// (bit-identical to the reference for finite data), EXACT=false uses FFMA (<= 1 ulp per step).
// Border pixels: TMA zero-fills out-of-range coordinates; for replicate / mirror / wrap (and for the
// ragged right edge when cols % 8 != 0) the few out-of-range stage entries are patched with
// resolveIndex()-ed global loads before the horizontal pass (reference border.zig:46-63), so the
// filter code itself has no border branches.
#include "zb_conv.h"
#include "zb_device.cuh"
#include "zb_shard.h"
#include "zb_tma.cuh"

namespace zb {

namespace {

constexpr int TW = 256;                  // strip width in pixels
constexpr int CHUNK = 8;                 // rows per pipeline step
constexpr int G = TW / 8 + 2;            // 8-pixel groups per stage row (one halo group each side)
constexpr int STAGE_BYTES = G * CHUNK * 128;          // 34816
constexpr int RING_ROWS = 24;
constexpr int RING_ROW_BYTES = TW * 16;               // 4096
constexpr int RING_BYTES = RING_ROWS * RING_ROW_BYTES;  // 98304
constexpr int NTHREADS = 256;
constexpr int MAX_HALF = 8;
constexpr int MAXK = 2 * MAX_HALF + 1;
// TMA ring depth: at 8192 x 8192, 15 taps, .mirror on an H100 SXM (700 W) 3 stages took 0.785 ms against 0.778 ms for 2 (sharded: 0.462 / 0.435)
constexpr int STAGES = 2;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + RING_BYTES + 64 + 1024;

struct FusedParams {
    float kx[MAXK];
    float ky[MAXK];
    const float4* src;
    float4* dst;
    unsigned long long src_pitch_px, dst_pitch_px;
    int rows, cols, border;
    int ngroups;     // floor(cols / 8): pixel groups the tensor map covers
    int n_strips;    // TW-pixel strips
    int n_units;     // work units: (row segment, strip) pairs, decoded by unit_at()
    int strip_lo, strip_hi;      // inner strips [strip_lo, strip_hi); the others are edge strips (their stages need x-border fixups)
    int n_segs, seg_chunks, seg_extra;   // inner strips: row segment s of [row0, row1) holds seg_chunks + (s < seg_extra) chunks
    int e_segs, e_chunks, e_extra;       // edge strips: the same, cut on their own
    int row0, row1;  // output rows this launch produces: [row0, row1) (the whole image unless the host pipeline slices it)
    int fix_rows;    // 1 if out-of-range rows need patching (border != zero)
    int fix_left;    // 1 if x < 0 needs patching
    int fix_right;   // 1 if x >= 8*ngroups needs patching (border != zero or ragged edge)
    int tma_row_off; // row of the tensor map that holds image row 0 (sharded blocks: the map starts at the first halo row)
    int edge_fast;   // .replicate / .mirror with cols % 8 == 0: the 8 columns left of x = 0 and right of x = cols - 1 are copies of
                     // columns TMA delivered into the same stage; lsrc / rsrc (host-resolved) say which
    int lsrc[8];     // stage pixel index the halo pixel x = e - 8 of the FIRST strip is copied from
    int rsrc[8];     // image column the halo pixel x = cols + e of the last strip is copied from
};

// Sharded launch (zb_shard_conv_separable): this rank holds one row block of a taller image, stored with `halo_cap` (>= CHUNK)
// spare rows above and below it.  The rows beyond the block are not border pixels but the neighbours' edge rows.  The kernel
// fetches them itself: in a prologue every CTA copies a slice of the 2 x half neighbour rows from the neighbours' memory (IPC
// mappings over NVLink; plain 128-bit loads, many in flight per thread) into the block's own halo rows, after which the ordinary
// TMA pipeline reads them like any other row.  (A TMA load straight from peer memory was measured first: 34 KB per chunk arrived in
// ~45 us -- the TMA unit keeps too few requests in flight for NVLink's latency -- which cost the whole step 47 us.)  The bands next
// to a neighbour are processed LAST, so nothing ever waits for the copy; the kernel also carries the whole synchronisation
// (ready / done flags, zb_shard.h).
struct ShardParams {
    const float4* up_rows;     // the upper neighbour's last `half` rows (null: global top edge, border mode applies)
    const float4* down_rows;   // the lower neighbour's first `half` rows (null: global bottom edge)
    unsigned long long up_pitch_px, down_pitch_px;
    int half;
    ShardLink link;
};

// Strip and output rows [ra, rb) of unit u.  Units [0, n_segs x inner strips) are the inner strips, segment-major (concurrent
// CTAs cover neighbouring strips of one segment); the edge strips' units follow.  ROTATE (sharded kernel, which has no edge class):
// segment s + 1 first, segment 0 -- the bands next to the neighbours -- last.
template <bool ROTATE>
__device__ __forceinline__ void unit_at(const FusedParams& p, int u, int& strip, int& ra, int& rb) {
    const int n_inner = p.strip_hi - p.strip_lo;
    int seg, chunks, extra;
    if (u < p.n_segs * n_inner) {
        seg = u / n_inner;
        strip = p.strip_lo + (u - seg * n_inner);
        if constexpr (ROTATE) seg = seg + 1 == p.n_segs ? 0 : seg + 1;
        chunks = p.seg_chunks;
        extra = p.seg_extra;
    } else {
        const int n_edge = p.n_strips - n_inner;
        u -= p.n_segs * n_inner;
        seg = u / n_edge;
        const int e = u - seg * n_edge;
        strip = e < p.strip_lo ? e : e - p.strip_lo + p.strip_hi;
        chunks = p.e_chunks;
        extra = p.e_extra;
    }
    ra = p.row0 + (seg * chunks + min(seg, extra)) * CHUNK;
    rb = min(ra + (chunks + (seg < extra ? 1 : 0)) * CHUNK, p.row1);
}

template <bool EXACT>
__device__ __forceinline__ void mac4(float4& acc, const float4& v, float k) {
    if constexpr (EXACT) {
        acc.x = __fadd_rn(acc.x, __fmul_rn(v.x, k));
        acc.y = __fadd_rn(acc.y, __fmul_rn(v.y, k));
        acc.z = __fadd_rn(acc.z, __fmul_rn(v.z, k));
        acc.w = __fadd_rn(acc.w, __fmul_rn(v.w, k));
    } else {
        acc.x = fmaf(v.x, k, acc.x);
        acc.y = fmaf(v.y, k, acc.y);
        acc.z = fmaf(v.z, k, acc.z);
        acc.w = fmaf(v.w, k, acc.w);
    }
}

// Patch the stage entries TMA could not provide (out-of-range rows / columns) per the border mode.
// Column patches of in-range rows are sourced from the stage itself whenever the resolved column is one
// TMA delivered (always the case for mirror / replicate): no global-memory latency on the per-chunk path
// of the edge strips.  Out-of-range rows (image top / bottom only) are fetched from global memory.
template <bool SHARD>
__device__ __noinline__ void fixup_stage(uint32_t stage, int y0, int xs0, bool fix_x, bool fix_rows, const FusedParams& p,
                                         int nb_lo, int nb_hi) {   // SHARD: rows in [nb_lo, 0) / [rows, nb_hi) are neighbour rows
    const int xlimit = p.ngroups * 8;
    auto stage_addr = [&](int rr, int xx) {
        const uint32_t line = (uint32_t)(rr * G + (xx >> 3));
        return stage + line * 128 + ((((uint32_t)xx & 7u) ^ (line & 7u)) << 4);
    };
    if (fix_x && p.edge_fast) {
        // .replicate / .mirror with cols % 8 == 0 (the usual case): the 8 columns either side of the image are 16-byte copies inside
        // the stage from the columns the host resolved (FusedParams::lsrc / rsrc) -- 8 rows x 8 columns per side, no index
        // arithmetic, no divisions.  It lives in this out-of-line function on purpose.  Of the 33 us the border costs per launch at
        // 8192 x 8192 (.mirror 0.436 ms, .zero 0.403) the patch LOOP is the small part (this version: -3 us); the rest is the call and
        // the extra barrier per chunk of an edge strip.  Both attempts to avoid them -- the same copies inlined into the chunk loop,
        // and the owner thread of each row copying its halo pixels right before reading them (no barrier at all) -- removed 20 us of
        // border cost and added 19-27 us to EVERY border mode: the loop's code grew by 50-100 instructions and 10-14 registers and
        // the kernel, FP32-issue bound with 1920 FFMAs per chunk, lost more in the steady state than it won at the edges.
        fix_x = false;
        if (threadIdx.x < 128) {
            const int side = threadIdx.x >> 6, rr = (threadIdx.x >> 3) & 7, e = threadIdx.x & 7;
            const int y = y0 + rr;
            bool row_ok = y >= 0 && y < p.rows;                  // rows beyond the image are rebuilt whole by the row pass
            if constexpr (SHARD) row_ok = row_ok || (y < 0 && y >= nb_lo) || (y >= p.rows && y < nb_hi);   // neighbour rows are real rows
            const bool edge = side == 0 ? xs0 < 0 : xs0 + G * 8 > p.cols;
            if (row_ok && edge) {
                const int s_dst = side == 0 ? e : p.cols - xs0 + e;
                const int s_src = side == 0 ? p.lsrc[e] : p.rsrc[e] - xs0;
                if (s_dst < G * 8) sts128(stage_addr(rr, s_dst), lds128(stage_addr(rr, s_src)));
            }
        }
    }
    if (fix_x) {
        const int nleft = xs0 < 0 ? min(-xs0, G * 8) : 0;                      // entries [0, nleft) have x < 0
        const int r0 = max(0, xlimit - xs0);                                    // first entry with x >= xlimit
        const int r1 = min(G * 8, p.cols - xs0 + MAX_HALF);                     // entries beyond cols + MAX_HALF are never read
        const int per_row = nleft + max(0, r1 - r0);
        for (int idx = threadIdx.x; idx < CHUNK * per_row; idx += NTHREADS) {
            const int rr = idx / per_row, e = idx - rr * per_row;
            const int xx = e < nleft ? e : r0 + (e - nleft);
            const int y = y0 + rr, x = xs0 + xx;
            const float4* rowp = p.src + (long long)y * (long long)p.src_pitch_px;
            if (y < 0 || y >= p.rows) {
                if constexpr (SHARD) {   // a neighbour's row: it sits in this block's halo rows (the prologue copied it)
                    if (y < nb_lo || y >= nb_hi) continue;
                } else {
                    continue;                                                   // handled by the row pass below
                }
            }
            const int rx = resolve_index(x, p.cols, p.border);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (rx >= 0) {
                const int sx = rx - xs0;
                if (rx < xlimit && sx >= 0 && sx < G * 8) v = lds128(stage_addr(rr, sx));   // delivered by TMA into this stage
                else v = __ldg(rowp + rx);
            }
            sts128(stage_addr(rr, xx), v);
        }
    }
    if (fix_rows) {
        for (int idx = threadIdx.x; idx < CHUNK * G * 8; idx += NTHREADS) {
            const int rr = idx / (G * 8);
            const int xx = idx - rr * (G * 8);
            const int y = y0 + rr, x = xs0 + xx;
            if (y >= 0 && y < p.rows) continue;
            if constexpr (SHARD) {
                if (y >= nb_lo && y < nb_hi) continue;   // neighbour rows: not border pixels
            }
            const int ry = resolve_index(y, p.rows, p.border);
            const int rx = resolve_index(x, p.cols, p.border);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ry >= 0 && rx >= 0) v = __ldg(p.src + (size_t)ry * p.src_pitch_px + rx);
            sts128(stage_addr(rr, xx), v);
        }
    }
}

// Vertical pass of one chunk: 8 output rows from ring rows [SLOT*8 + 8-HALF, SLOT*8 + 16+HALF) (mod 24).
template <int HALF, bool EXACT, int SLOT>
__device__ __forceinline__ void v_pass(uint32_t v_col, const FusedParams& p, float4* out, bool col_ok, int rows_left) {
    constexpr int K = 2 * HALF + 1;
    constexpr int NLOAD = CHUNK + 2 * HALF;
    float4 acc[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < NLOAD; ++j) {
        const int sr = (SLOT * CHUNK + 8 - HALF + j) % RING_ROWS;
        const float4 v = lds128(v_col + (uint32_t)(sr * RING_ROW_BYTES));
#pragma unroll
        for (int o = 0; o < 8; ++o) {
            const int ti = j - o;
            if (ti >= 0 && ti < K) mac4<EXACT>(acc[o], v, p.ky[ti]);
        }
    }
    if (col_ok) {
#pragma unroll
        for (int o = 0; o < 8; ++o)
            if (o < rows_left) __stcs(out + (size_t)o * p.dst_pitch_px, acc[o]);
    }
}

// The heavy part of the kernel: this CTA's units k_begin <= k < k_end (unit = blockIdx.x + k * gridDim.x), TMA pipeline filled at
// entry and drained at exit; `count0` = chunks this CTA has consumed before (stage index and mbarrier parity carry on from there).
// Returns the updated count.  nbr (SHARD): bit 0 = the rows above the block are the upper neighbour's (already in the halo rows),
// bit 1 = the rows below are the lower neighbour's.
template <int HALF, bool EXACT, bool SHARD>
__device__ __forceinline__ uint32_t fused_units(const CUtensorMap& tmap, const FusedParams& p, unsigned nbr, int k_begin, int k_end, uint32_t count0) {
    constexpr int K = 2 * HALF + 1;
    constexpr int NLOAD = CHUNK + 2 * HALF;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t ring = smem0 + STAGES * STAGE_BYTES;
    const uint32_t bar0 = ring + RING_BYTES;

    const int tid = threadIdx.x;
    const long long u_first = (long long)blockIdx.x + (long long)k_begin * gridDim.x;
    const long long u_last = (long long)blockIdx.x + (long long)k_end * gridDim.x;
    const int n_units = (int)min((long long)p.n_units, u_last);
    if (u_first >= n_units) return count0;
    // does a chunk of rows [y, y + CHUNK) read neighbour rows?
    auto touches_neighbour = [&](int y) { return ((nbr & 1u) && y < 0) || ((nbr & 2u) && y + CHUNK > p.rows); };

    // ---- producer (thread 0): a cursor over this CTA's (unit, chunk) sequence, STAGES chunks ahead ----
    int pu = (int)u_first, pi = 0;
    uint32_t pcount = count0;
    auto produce = [&]() {
        if (pu >= n_units) return;
        int strip, ra, rb;
        unit_at<SHARD>(p, pu, strip, ra, rb);
        const int n_in = (rb - ra + CHUNK - 1) / CHUNK + 2;
        const uint32_t st = pcount % STAGES;
        const int y = ra - CHUNK + CHUNK * pi;
        fence_proxy_async();
        mbar_arrive_expect_tx(bar0 + 8 * st, STAGE_BYTES);
        tma_load_3d(smem0 + st * STAGE_BYTES, &tmap, 0, strip * (TW / 8) - 1, y + p.tma_row_off, bar0 + 8 * st);
        ++pcount;
        if (++pi == n_in) { pi = 0; pu += gridDim.x; }
    };
    if (tid == 0)
        for (int i = 0; i < STAGES; ++i) produce();

    // H-pass role: lane -> pixel group (8 consecutive pixels), warp -> row of the chunk
    const int ht = tid & 31, hr = tid >> 5;
    // V-pass role: thread -> pixel column, 8 consecutive output rows
    const int vx = tid;
    const uint32_t v_col = ring + (uint32_t)(vx >> 3) * 128u + ((((uint32_t)vx & 7u) ^ (((uint32_t)vx >> 3) & 7u)) << 4);
    const uint32_t h_ring_col = ring + (uint32_t)ht * 128u;
    const uint32_t h_key = (uint32_t)ht & 7u;

    uint32_t ccount = count0;  // chunks consumed by this CTA

    for (int unit = (int)u_first; unit < n_units; unit += gridDim.x) {
        int strip, ra, rb;
        unit_at<SHARD>(p, unit, strip, ra, rb);
        const int x0 = strip * TW;
        const int n_out = (rb - ra + CHUNK - 1) / CHUNK;  // output chunks
        const int n_in = n_out + 2;                       // input chunks: chunk i covers rows [ra-8+8i, ra+8i)
        const int g0 = x0 / 8 - 1;

        for (int i = 0; i < n_in; ++i, ++ccount) {
            const uint32_t st = ccount % STAGES;
            const uint32_t stage = smem0 + st * STAGE_BYTES;
            while (!mbar_try_wait(bar0 + 8 * st, (ccount / STAGES) & 1u)) {}
            const int y0 = ra - CHUNK + CHUNK * i;
            bool fix_r = p.fix_rows && (y0 < 0 || y0 + CHUNK > p.rows);
            if constexpr (SHARD) {   // rows beyond the block on a neighbour side are real rows (already in the halo), not border pixels
                if (touches_neighbour(y0)) fix_r = false;
            }
            const bool fix_x = (p.fix_left && g0 < 0) || (p.fix_right && (g0 + G) * 8 > p.ngroups * 8);
            if (fix_r || fix_x) {
                fixup_stage<SHARD>(stage, y0, g0 * 8, fix_x, fix_r, p, (nbr & 1u) ? INT_MIN : 0, (nbr & 2u) ? INT_MAX : p.rows);
                __syncthreads();
            }

            // ---------------- H(i): stage -> ring rows [(i%3)*8, +8) ----------------
            {
                const uint32_t line0 = (uint32_t)(hr * G + ht);
                // address of pixel c of stage line l = base(l) ^ (c << 4), base(l) = stage + l*128 + ((l & 7) << 4)  (stage is 1 KB aligned)
                uint32_t lbase[3];
#pragma unroll
                for (int l = 0; l < 3; ++l) lbase[l] = stage + (line0 + l) * 128u + (((line0 + l) & 7u) << 4);
                const uint32_t rrow = h_ring_col + (uint32_t)(((i % 3) * CHUNK + hr) * RING_ROW_BYTES);
                float4 acc[8];
#pragma unroll
                for (int o = 0; o < 8; ++o) acc[o] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int j = 0; j < NLOAD; ++j) {
                    const int pidx = 8 - HALF + j;  // pixel index relative to the start of group `ht` of the stage row
                    const float4 v = lds128(lbase[pidx >> 3] ^ (((uint32_t)pidx & 7u) << 4));
#pragma unroll
                    for (int o = 0; o < 8; ++o) {
                        const int ti = j - o;
                        if (ti >= 0 && ti < K) mac4<EXACT>(acc[o], v, p.kx[ti]);
                    }
                }
#pragma unroll
                for (int o = 0; o < 8; ++o) sts128(rrow + ((((uint32_t)o) ^ h_key) << 4), acc[o]);
            }
            __syncthreads();  // ring slot complete; stage `st` is free again

            if (tid == 0) produce();  // refill the stage just drained (the chunk STAGES ahead, possibly of the next unit)

            // ---------------- V(i-2): ring -> global rows [ra+8c, ra+8c+8) ----------------
            if (i >= 2) {
                const int c = i - 2;
                const int x = x0 + vx;
                const int yb = ra + CHUNK * c;
                float4* out = p.dst + (size_t)yb * p.dst_pitch_px + x;
                const bool col_ok = x < p.cols;
                switch (c % 3) {  // the ring slot of chunk c is compile-time inside each case: loads use immediate offsets
                    case 0: v_pass<HALF, EXACT, 0>(v_col, p, out, col_ok, rb - yb); break;
                    case 1: v_pass<HALF, EXACT, 1>(v_col, p, out, col_ok, rb - yb); break;
                    default: v_pass<HALF, EXACT, 2>(v_col, p, out, col_ok, rb - yb); break;
                }
            }
            __syncthreads();  // V(i-2) done reading the slot H(i+1) will overwrite
        }
    }
    return ccount;
}

template <int HALF, bool EXACT, bool SHARD>
__device__ __forceinline__ void fused_sep_rgbaf32_body(const CUtensorMap& tmap, const FusedParams& p, const ShardParams* sp) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar0 = smem0 + STAGES * STAGE_BYTES + RING_BYTES;
    const int tid = threadIdx.x;
    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap) : "memory");
        for (int i = 0; i < STAGES; ++i) mbar_init(bar0 + 8 * i, 1);
        fence_barrier_init();
    }
    if constexpr (!SHARD) {
        __syncthreads();
        fused_units<HALF, EXACT, false>(tmap, p, 0u, 0, INT_MAX / 2048, 0u);
    } else {
        ShardCtrl* me = sp->link.self;
        const unsigned long long epoch = sp->link.epoch;
        const unsigned nbr = (sp->up_rows ? 1u : 0u) | (sp->down_rows ? 2u : 0u);
        // ---- prologue: the CTAs with a slice of the neighbours' edge rows copy it into my halo rows (plain loads over NVLink, all
        // issued before the first use so the round trips overlap); the others go straight to their rows ----
        const int per_side = sp->half * p.cols;                      // pixels
        const int total = (sp->up_rows ? per_side : 0) + (sp->down_rows ? per_side : 0);
        constexpr int BATCH = 12;   // loads in flight per thread: the copy is a handful of NVLink round trips, not a bandwidth problem
        // The copy is done by the CTAs with the lightest load: units are dealt round robin, so CTAs [rem, grid) have one unit less
        // than the others (the host launches a full grid even when there are fewer units than SMs: those CTAs have none), which is
        // far more slack than the copy needs.  rem == 0: everyone carries the same load and shares the copy.
        const int rem = p.n_units % (int)gridDim.x;
        const int n_copiers = (int)gridDim.x - rem;
        const int ci = (int)blockIdx.x - rem;
        const bool copier = ci >= 0 && (long long)ci * NTHREADS * BATCH < total;
        if (tid == 0) {
            // this kernel is stream-ordered after whatever produced my source block: tell the neighbours it is complete; a CTA that
            // reads their rows waits until theirs are
            if (blockIdx.x == 0) {
                me->dbg[0] = global_timer_ns();
                if (sp->link.up) st_release_sys(&sp->link.up->ready_from[1], epoch);
                if (sp->link.down) st_release_sys(&sp->link.down->ready_from[0], epoch);
            }
            if (copier) {
                if (sp->up_rows) shard_wait_ge(&me->ready_from[0], epoch, me);
                if (sp->down_rows) shard_wait_ge(&me->ready_from[1], epoch, me);
                if (ci == 0) me->dbg[1] = global_timer_ns();
            }
        }
        __syncthreads();
        if (copier) {
            for (int base = ci * NTHREADS * BATCH; base < total; base += n_copiers * NTHREADS * BATCH) {
                float4 v[BATCH];
                float4* dstp[BATCH];
    #pragma unroll
                for (int k = 0; k < BATCH; ++k) {
                    int e = base + k * NTHREADS + tid;
                    dstp[k] = nullptr;
                    if (e < total) {
                        const bool upper = sp->up_rows && e < per_side;
                        if (!upper && sp->up_rows) e -= per_side;
                        const int r = e / p.cols, x = e - r * p.cols;
                        if (upper) {
                            v[k] = *(sp->up_rows + (size_t)r * sp->up_pitch_px + x);
                            dstp[k] = const_cast<float4*>(p.src) + (long long)(r - sp->half) * (long long)p.src_pitch_px + x;
                        } else {
                            v[k] = *(sp->down_rows + (size_t)r * sp->down_pitch_px + x);
                            dstp[k] = const_cast<float4*>(p.src) + (long long)(p.rows + r) * (long long)p.src_pitch_px + x;
                        }
                    }
                }
    #pragma unroll
                for (int k = 0; k < BATCH; ++k)
                    if (dstp[k]) *dstp[k] = v[k];
            }
            asm volatile("fence.proxy.async;" ::: "memory");   // these generic-proxy stores are read by TMA (async proxy) later on
            __syncthreads();
        }
        if (tid == 0) {
            __threadfence();
            if (atomicAdd(&me->halo_reads[0], 1u) == gridDim.x - 1u) {   // every CTA's slice has landed
                me->halo_reads[0] = 0;
                me->dbg[2] = global_timer_ns();
                __threadfence();
                st_release_sys(&me->halo_landed, epoch);
                // the neighbours' rows have been read: they may overwrite their source again
                if (sp->up_rows) st_release_sys(&sp->link.up->done_from[1], epoch);
                if (sp->down_rows) st_release_sys(&sp->link.down->done_from[0], epoch);
            }
        }
        // ---- the rows: first the units that read no halo row, then -- once every CTA's copy has landed (normally long ago) -- the
        // two bands next to the neighbours, which the unit order puts last ----
        // The unit loop is inlined twice with the wait for the halo rows in between.  With a spin loop anywhere INSIDE the loop
        // ptxas stops keeping the 30 taps in uniform registers and reloads them from the constant bank in every H and V pass (0.50 ms
        // against 0.44 ms for the same rows); behind a real call the taps arrive through a generic pointer and every FFMA takes three
        // vector registers.
        const long long first_halo_unit = (long long)max(0, p.n_segs - 2) * p.n_strips;
        const int k_split = first_halo_unit <= (long long)blockIdx.x ? 0 : (int)((first_halo_unit - blockIdx.x + gridDim.x - 1) / gridDim.x);
        const uint32_t count = fused_units<HALF, EXACT, true>(tmap, p, nbr, 0, k_split, 0u);
        if ((long long)blockIdx.x + (long long)k_split * gridDim.x < (long long)p.n_units) {   // this CTA has halo units
            if (tid == 0) {
                shard_wait_ge(&me->halo_landed, epoch, me);
                asm volatile("fence.proxy.async;" ::: "memory");   // the acquire above orders TMA's (async proxy) reads of the halo rows
            }
            __syncthreads();
            fused_units<HALF, EXACT, true>(tmap, p, nbr, k_split, INT_MAX / 2048, count);
        }
        // The kernel may not complete before both neighbours have finished reading this block's edge rows: whatever runs
        // next on this stream is then free to overwrite the source.  The last CTA to leave does the waiting.
        if (tid == 0) {
            ShardCtrl* me = sp->link.self;
            __threadfence();
            if (atomicAdd(&me->exit_ticket, 1u) == gridDim.x - 1u) {
                me->exit_ticket = 0;
                me->dbg[3] = global_timer_ns();
                if (sp->link.up) shard_wait_ge(&me->done_from[0], sp->link.epoch, me);
                if (sp->link.down) shard_wait_ge(&me->done_from[1], sp->link.epoch, me);
                me->dbg[4] = global_timer_ns();
            }
        }
    }
}


template <int HALF, bool EXACT>
__global__ void __launch_bounds__(NTHREADS, 1)
fused_sep_rgbaf32_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ FusedParams p) {
    fused_sep_rgbaf32_body<HALF, EXACT, false>(tmap, p, nullptr);
}

template <int HALF, bool EXACT>
__global__ void __launch_bounds__(NTHREADS, 1)
fused_sep_rgbaf32_shard_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ FusedParams p,
                               const __grid_constant__ ShardParams sp) {
    fused_sep_rgbaf32_body<HALF, EXACT, true>(tmap, p, &sp);
}

// sp: the sharded kernel's parameters (null: the single-GPU kernel)
template <int HALF>
int launch_fused(const CUtensorMap& tmap, const FusedParams& p, const ShardParams* sp, int grid, bool exact, cudaStream_t s) {
    if (sp) {
        auto k = exact ? fused_sep_rgbaf32_shard_kernel<HALF, true> : fused_sep_rgbaf32_shard_kernel<HALF, false>;
        ZB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));  // per device; cheap
        k<<<grid, NTHREADS, SMEM_BYTES, s>>>(tmap, p, *sp);
    } else {
        auto k = exact ? fused_sep_rgbaf32_kernel<HALF, true> : fused_sep_rgbaf32_kernel<HALF, false>;
        ZB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        k<<<grid, NTHREADS, SMEM_BYTES, s>>>(tmap, p);
    }
    ZB_LAUNCHED();
    return ZB_OK;
}

int launch_half(int half, const CUtensorMap& tmap, const FusedParams& p, const ShardParams* sp, int grid, bool exact, cudaStream_t s) {
    switch (half) {
        case 1: return launch_fused<1>(tmap, p, sp, grid, exact, s);
        case 2: return launch_fused<2>(tmap, p, sp, grid, exact, s);
        case 3: return launch_fused<3>(tmap, p, sp, grid, exact, s);
        case 4: return launch_fused<4>(tmap, p, sp, grid, exact, s);
        case 5: return launch_fused<5>(tmap, p, sp, grid, exact, s);
        case 6: return launch_fused<6>(tmap, p, sp, grid, exact, s);
        case 7: return launch_fused<7>(tmap, p, sp, grid, exact, s);
        case 8: return launch_fused<8>(tmap, p, sp, grid, exact, s);
    }
    return ZB_ERR_UNSUPPORTED;
}

}  // namespace

// Tensor map of one row block of RGBA f32 pixels: {32 floats = 8 px, groups, rows}, box {8 px, G groups, CHUNK rows}.
static int encode_block_map(EncodeTiledFn encode, CUtensorMap& tmap, void* data, int ngroups, int rows, uint64_t stride_px) {
    const cuuint64_t gdim[3] = {32, (cuuint64_t)ngroups, (cuuint64_t)rows};
    const cuuint64_t gstr[2] = {128, (cuuint64_t)stride_px * 16};
    const cuuint32_t box[3] = {32, (cuuint32_t)G, (cuuint32_t)CHUNK};
    const cuuint32_t estr[3] = {1, 1, 1};
    CUresult cr = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, data, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
        snprintf(t_last_error, sizeof(t_last_error), "cuTensorMapEncodeTiled failed: %d", (int)cr);
        return ZB_ERR_UNSUPPORTED;
    }
    return ZB_OK;
}

// A chunk of an edge strip (one whose stages need x-border fixups) costs its CTA about 5/4 of an inner strip's chunk: the
// fixup_stage() call and one more barrier.  Measured on an H100 SXM (700 W) at 8192 x 8192, 15 taps, .mirror, every strip cut into
// 4 segments of 2048 rows: 0.932 ms, against 0.782 ms for .zero (no edge strips) -- the 8 edge CTAs set the kernel time.
constexpr long long EDGE_COST_NUM = 5, EDGE_COST_DEN = 4;

// Work plan of the single-GPU kernels: the inner strips are cut into P row segments, the edge strips into E >= P, one unit per
// (segment, strip), dealt round robin to min(units, SMs) persistent CTAs.  A unit of c chunks costs its CTA c + 2 pipeline steps
// (two halo chunks), so the plan minimises the busiest CTA's steps, waves x max(ceil(C / P) + 2, 5/4 x (ceil(C / E) + 2)) with
// C = ceil(nrows / CHUNK), where E takes the CTAs the inner units leave free in their waves; ties go to fewer units (fewer halo
// rows).  Segments differ by at most one chunk and hold at least 8 chunks (64 rows): each halo chunk is a second DRAM read of rows
// the neighbouring segment reads.  With one unit per CTA all CTAs start together, so neighbouring inner strips stay in lockstep
// and their x-halos stay L2 hits.  8192 x 8192 on 132 SMs, .mirror: 30 inner strips x 4 segments of 2048 rows (258 steps) and
// 2 edge strips x 6 segments of 1368 / 1360 rows (173 steps, ~216 weighted) on 132 CTAs; 256-row bands dealt round robin (1024
// units on 132 CTAs) cost the busiest CTA 8 x 34 = 272 steps.  A 256-row window of the host pipeline: 4 segments of 64 rows.
static void plan_units(int nrows, int sm_count, FusedParams& p) {
    const long long chunks = (nrows + CHUNK - 1) / CHUNK;
    const long long max_segs = chunks / 8 < 1 ? 1 : (chunks / 8 < sm_count ? chunks / 8 : sm_count);
    const long long n_inner = p.strip_hi - p.strip_lo, n_edge = p.n_strips - n_inner;
    auto steps = [&](long long segs) { return (chunks + segs - 1) / segs + 2; };
    long long best_cost = -1, best_units = 0, best_s = 1, best_e = 1;
    for (long long s = 1; s <= max_segs; ++s) {
        const long long waves = (s * p.n_strips + sm_count - 1) / sm_count;
        long long e = s;
        if (n_edge > 0) {
            long long e_max = (waves * sm_count - s * n_inner) / n_edge;
            if (e_max > max_segs) e_max = max_segs;
            while (e < e_max && EDGE_COST_NUM * steps(e) > EDGE_COST_DEN * steps(s)) ++e;
        }
        const long long inner = n_inner > 0 ? EDGE_COST_DEN * steps(s) : 0, edge = n_edge > 0 ? EDGE_COST_NUM * steps(e) : 0;
        const long long cost = waves * (inner > edge ? inner : edge), units = s * n_inner + e * n_edge;
        if (best_cost < 0 || cost < best_cost || (cost == best_cost && units < best_units)) {
            best_cost = cost;
            best_units = units;
            best_s = s;
            best_e = e;
        }
    }
    p.n_units = (int)best_units;
    p.n_segs = (int)best_s;
    p.seg_chunks = (int)(chunks / best_s);
    p.seg_extra = (int)(chunks % best_s);
    p.e_segs = (int)best_e;
    p.e_chunks = (int)(chunks / best_e);
    p.e_extra = (int)(chunks % best_e);
}

// Validates the call, fills the kernel parameters and encodes the tensor map of `src`.  `bands`: the sharded kernel's plan (bands of
// about conv.band_rows rows, all seg_chunks long but the last, several per CTA) instead of plan_units().
static int fused_prepare(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border, int row0, int row1,
                         bool bands, FusedParams& p, CUtensorMap& tmap, int& grid, int& half_out, EncodeTiledFn& encode) {
    const int half_x = nx / 2, half_y = ny / 2;
    const int half = half_x > half_y ? half_x : half_y;
    if (half < 1 || half > MAX_HALF) return ZB_ERR_UNSUPPORTED;
    if (src->cols < 16 || src->rows < 16) return ZB_ERR_UNSUPPORTED;  // tiny images: generic path
    if (images_overlap(src, dst, 16)) return ZB_ERR_UNSUPPORTED;       // in place / overlapping views: generic path (temp plane)
    if (((uintptr_t)src->data & 15u) || ((uintptr_t)dst->data & 15u)) return ZB_ERR_UNSUPPORTED;
    // taps with |k| < 1e-10 are skipped by the reference only in the interior (convolution.zig:459-467): generic path
    for (int i = 0; i < nx; ++i) if (fabsf(kx[i]) < 1e-10f) return ZB_ERR_UNSUPPORTED;
    for (int i = 0; i < ny; ++i) if (fabsf(ky[i]) < 1e-10f) return ZB_ERR_UNSUPPORTED;
    encode = encode_tiled_fn();
    if (!encode) return ZB_ERR_UNSUPPORTED;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    if (di.smem_optin < (size_t)SMEM_BYTES) return ZB_ERR_UNSUPPORTED;

    memset(&p, 0, sizeof(p));
    // tap i of an n-tap kernel acts at offset i - n/2 (convolution.zig:527,542): place it at index i + (half - n/2)
    for (int i = 0; i < nx; ++i) p.kx[i + (half - half_x)] = kx[i];
    for (int i = 0; i < ny; ++i) p.ky[i + (half - half_y)] = ky[i];
    p.src = (const float4*)src->data;
    p.dst = (float4*)dst->data;
    p.src_pitch_px = src->stride;
    p.dst_pitch_px = dst->stride;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.border = border;
    p.ngroups = p.cols / 8;
    p.n_strips = (p.cols + TW - 1) / TW;
    p.row0 = row0 < 0 ? 0 : row0;
    p.row1 = (row1 < 0 || row1 > p.rows) ? p.rows : row1;
    if (p.row1 <= p.row0) { grid = 0; return ZB_OK; }
    const int nrows = p.row1 - p.row0;
    p.fix_rows = border != ZB_BORDER_ZERO;
    p.fix_left = border != ZB_BORDER_ZERO;
    p.fix_right = (border != ZB_BORDER_ZERO) || (p.cols % 8 != 0);
    p.strip_lo = 0;
    p.strip_hi = p.n_strips;
    if (bands) {
        const BandPlan plan = plan_bands(nrows, p.n_strips, di.sm_count, g_tune_band_rows.load());
        p.n_segs = plan.n_bands;
        p.seg_chunks = plan.band_rows / CHUNK;
        p.n_units = p.n_segs * p.n_strips;
    } else {
        // edge strips: the stages fused_units() patches with fixup_stage() for x < 0 or x >= 8 * ngroups
        if (p.fix_left) p.strip_lo = 1;
        while (p.fix_right && p.strip_hi > p.strip_lo && (p.strip_hi - 1) * (TW / 8) - 1 + G > p.ngroups) --p.strip_hi;
        if (p.strip_hi <= p.strip_lo) { p.strip_lo = 0; p.strip_hi = p.n_strips; }   // every strip is an edge strip
        plan_units(nrows, di.sm_count, p);
    }
    p.edge_fast = g_tune_edge_fast.load() && (border == ZB_BORDER_REPLICATE || border == ZB_BORDER_MIRROR) && p.cols % 8 == 0 && p.cols >= 16;
    for (int e = 0; e < 8; ++e) {   // border.zig:46-63 resolveIndex for the 8 columns either side (replicate; mirror = reflect-101)
        const int xl = e - 8, xr = p.cols + e;
        p.lsrc[e] = 8 + (border == ZB_BORDER_REPLICATE ? 0 : -xl);
        p.rsrc[e] = border == ZB_BORDER_REPLICATE ? p.cols - 1 : 2 * (p.cols - 1) - xr;
    }

    if ((rc = encode_block_map(encode, tmap, src->data, p.ngroups, p.rows, src->stride))) return rc;
    grid = p.n_units < di.sm_count ? p.n_units : di.sm_count;
    half_out = half;
    return ZB_OK;
}

int conv_separable_fused_rgbaf32(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border,
                                 bool exact, cudaStream_t s, int row0, int row1) {
    FusedParams p;
    CUtensorMap tmap;
    EncodeTiledFn encode;
    int grid = 0, half = 0;
    int rc = fused_prepare(src, dst, kx, nx, ky, ny, border, row0, row1, false, p, tmap, grid, half, encode);
    if (rc || grid == 0) return rc;
    t_last_kernel = exact ? "fused_sep_rgbaf32_exact" : "fused_sep_rgbaf32";
    return launch_half(half, tmap, p, nullptr, grid, exact, s);
}

// One launch per step: the convolution of this rank's row block of a taller image.  src must own `halo_cap` >= 8 rows of the same
// stride above and below the block; the kernel's prologue copies the neighbours' `half` edge rows into them over NVLink.
int conv_separable_fused_rgbaf32_shard(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border,
                                       bool exact, const PeerBlock& up, const PeerBlock& down, uint32_t halo_cap, const ShardLink& link,
                                       cudaStream_t s) {
    if (src->rows % CHUNK != 0 || halo_cap < (uint32_t)CHUNK) return ZB_ERR_UNSUPPORTED;   // chunks must not straddle the block
    FusedParams p;
    CUtensorMap tmap;
    EncodeTiledFn encode;
    int grid = 0, half = 0;
    int rc = fused_prepare(src, dst, kx, nx, ky, ny, border, 0, -1, true, p, tmap, grid, half, encode);
    if (rc) return rc;
    if (grid == 0) return ZB_ERR_UNSUPPORTED;
    const uint32_t hv = (uint32_t)(ny / 2);   // rows the vertical pass reaches into a neighbour
    if ((up.data && (up.rows < hv || ((uintptr_t)up.data & 15u))) || (down.data && (down.rows < hv || ((uintptr_t)down.data & 15u))))
        return ZB_ERR_UNSUPPORTED;
    // the tensor map spans the block AND its halo rows; the image's row 0 is the map's row halo_cap
    void* ext = (char*)src->data - (size_t)halo_cap * src->stride * 16;
    if ((rc = encode_block_map(encode, tmap, ext, p.ngroups, (int)(src->rows + 2 * halo_cap), src->stride))) return rc;
    p.tma_row_off = (int)halo_cap;
    p.fix_rows = 1;   // beyond a GLOBAL edge the halo rows hold no image data: every border mode (zero included) patches them
    ShardParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.half = (int)hv;
    if (up.data && hv) {
        sp.up_rows = (const float4*)up.data + (size_t)(up.rows - hv) * up.stride;
        sp.up_pitch_px = up.stride;
    }
    if (down.data && hv) {
        sp.down_rows = (const float4*)down.data;
        sp.down_pitch_px = down.stride;
    }
    sp.link = link;
    if (!sp.up_rows) sp.link.up = nullptr;
    if (!sp.down_rows) sp.link.down = nullptr;
    {   // always a full grid: CTAs beyond the unit count only copy halo rows (all CTAs are co-resident: one per SM)
        DeviceInfo di;
        if ((rc = device_info(&di))) return rc;
        grid = di.sm_count;
    }
    t_last_kernel = exact ? "fused_sep_rgbaf32_shard_exact" : "fused_sep_rgbaf32_shard";
    return launch_half(half, tmap, p, &sp, grid, exact, s);
}

}  // namespace zb
