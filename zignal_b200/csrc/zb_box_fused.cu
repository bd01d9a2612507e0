// zb_box_fused.cu -- Image.boxBlur / sharpen for 8-bit images without materialising the summed-area table in HBM.
//
// Reference: integral.zig:41-78 (f32 SAT: row prefix, then column accumulation), :85-90 (((D - left) - top) + corner),
// :194-269 / :325-422 (clipped-window box mean, 2*orig - blur), image.zig:635-648, :785-799.
//
// The SAT is f32 and its sums pass 2^24, so the SUMMATION ORDER is part of the result.  Two facts make a fused,
// parallel evaluation possible without changing a single bit:
//   * the row prefix P[r][c] = sum_{x<=c} src[r][x] of an 8-bit row is an integer < 2^24 (cols <= 65793): exact in f32,
//     so it may be computed in ANY order (integer warp scans);
//   * the column pass S[r][c] = fl(S[r-1][c] + P[r][c]) is a sequential chain in r, but chains of different columns are
//     independent, and a chain can be resumed from any row whose S is known.
// Three kernels (traffic: the source three times, the destination once, ~2% of it in side tables -- the 3-kernel SAT
// path moves 17x the image):
//   box_row_offsets : O[r][s] = exact integer row prefix at the first column of strip s          (one warp per row)
//   box_checkpoints : the only sequential pass, kept to the bare chain: one WARP per (strip, channel) walks all rows with
//                     no block-level synchronisation (unit loads run ahead, one warp scan per row) and stores S at the
//                     row above each band's first input row
//   box_chain       : one CTA per (strip, band): resumes the chains from its checkpoint, keeps the last 2r+2 SAT rows
//                     of its strip in a shared-memory ring and evaluates the box means / sharpen from it.
// Geometry: a "unit" is 4 bytes = one Rgba pixel (4 chains) or 4 gray pixels (1 chain each); a strip is 128 units =
// 512 element columns of which the inner OU = 128 - 2*MU units are outputs (MU covers radius+1 columns of halo).
#include "zb_device.cuh"
#include "zb_internal.h"

namespace zb {

namespace {

constexpr int SU = 128;          // units per strip row
constexpr int SE = 4 * SU;       // element columns per strip
constexpr int GR = 8;            // rows per block (one warp per row in the P phase)
constexpr int BF_THREADS = 256;
constexpr int BAND = 64;         // output rows per band

struct BoxParams {
    const uint8_t* src;
    uint8_t* dst;
    size_t src_pitch, dst_pitch;   // bytes
    int rows, cols;
    int row_units;                 // ceil(cols * CH / 4)
    int row_bytes;                 // cols * CH
    int radius, mu, ou, n_strips, n_bands;
    float c;                       // adaptive threshold: the constant subtracted from the mean
    int ring;                      // rows in the SAT ring (power of two)
    // both tables hold (prefix - 2^23) as f32 -- exact, since prefixes are integers below 2^24 -- so that
    // P = table + float(2^23 + small) needs no integer-to-float conversion in the consumers
    const float* offs;             // [rows][n_strips][4]   row prefix at each strip's first unit
    const float* offs32;           // [rows][n_win][4]      row prefix at every 32nd unit, channel order 0,2,1,3 (checkpoint pass)
    int n_win;                     // ceil(row_units / 32)
    int ck_pitch;                  // floats per checkpoint row: n_win * 128
    float* ckpt;                   // [n_bands][ck_pitch]   S at row (band * BAND - radius - 2), indexed by global element column
};

// 4 bytes of a row at unit `u` (0 outside the row; the last unit of a gray row may be partial, an Rgba unit never is)
template <int CH>
__device__ __forceinline__ uint32_t load_unit(const uint8_t* __restrict__ rowp, int u, int row_units, int row_bytes) {
    if ((unsigned)u >= (unsigned)row_units) return 0u;
    if (CH == 4 || 4 * u + 4 <= row_bytes) return __ldg(reinterpret_cast<const uint32_t*>(rowp) + u);
    uint32_t v = 0;
    for (int b = 0; 4 * u + b < row_bytes; ++b) v |= (uint32_t)rowp[4 * (size_t)u + b] << (8 * b);
    return v;
}

// P tile index with a 16-byte-chunk swizzle: the P phase stores 4 consecutive chunks per lane (64-byte stride between
// lanes), the chain phase reads consecutive floats; XOR-ing the chunk position with the low bits of its 128-byte group
// makes both conflict-free.
__device__ __forceinline__ int pt_chunk(int chunk) { return (chunk & ~7) | ((chunk ^ (chunk >> 3)) & 3) | (chunk & 4); }
__device__ __forceinline__ int pt_index(int e) { return pt_chunk(e >> 2) * 4 + (e & 3); }

// ---- 1. exact row prefixes: at every 32nd unit (for the checkpoint pass) and at every strip start ------------------------------
template <int CH>
__global__ void __launch_bounds__(256) box_row_offsets(const BoxParams p, float* __restrict__ offs, float* __restrict__ offs32) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (r >= p.rows) return;
    const uint8_t* rowp = p.src + (size_t)r * p.src_pitch;
    int4 carry = make_int4(0, 0, 0, 0);
    int s = 0;                       // next strip whose start has not been passed
    int next_start = -p.mu;          // unit index of strip s's first unit
    float4* out = reinterpret_cast<float4*>(offs) + (size_t)r * p.n_strips;
    float4* out32 = reinterpret_cast<float4*>(offs32) + (size_t)r * p.n_win;
    auto biased = [](int a, int b, int c, int d) {
        return make_float4((float)(a - 8388608), (float)(b - 8388608), (float)(c - 8388608), (float)(d - 8388608));
    };
    while (s < p.n_strips && next_start <= 0) {   // strips that start at or left of the row start: prefix 0
        if (lane == 0) out[s] = biased(carry.x, carry.y, carry.z, carry.w);
        ++s;
        next_start += p.ou;
    }
    for (int w = 0; w < p.n_win; ++w) {
        const int u0 = w * 32;
        const uint32_t v = load_unit<CH>(rowp, u0 + lane, p.row_units, p.row_bytes);
        int c[4];
        if constexpr (CH == 4) {
            c[0] = v & 0xFF; c[1] = (v >> 8) & 0xFF; c[2] = (v >> 16) & 0xFF; c[3] = v >> 24;
        } else {
            c[0] = (int)__dp4a(v, 0x01010101u, 0u); c[1] = c[2] = c[3] = 0;
        }
        if (lane == 0) out32[w] = biased(carry.x, carry.z, carry.y, carry.w);   // channel pairs {0,2} {1,3} contiguous
        if (s < p.n_strips && next_start < u0 + 32) {   // a strip starts inside this window (at most one: OU >= 96)
            const int pos = next_start - u0;              // exclusive prefix over lanes < pos
            int4 part = carry;
            part.x += __reduce_add_sync(0xffffffffu, lane < pos ? c[0] : 0);
            if constexpr (CH == 4) {
                part.y += __reduce_add_sync(0xffffffffu, lane < pos ? c[1] : 0);
                part.z += __reduce_add_sync(0xffffffffu, lane < pos ? c[2] : 0);
                part.w += __reduce_add_sync(0xffffffffu, lane < pos ? c[3] : 0);
            }
            if (lane == 0) out[s] = biased(part.x, part.y, part.z, part.w);
            ++s;
            next_start += p.ou;
        }
        carry.x += __reduce_add_sync(0xffffffffu, c[0]);
        if constexpr (CH == 4) {
            carry.y += __reduce_add_sync(0xffffffffu, c[1]);
            carry.z += __reduce_add_sync(0xffffffffu, c[2]);
            carry.w += __reduce_add_sync(0xffffffffu, c[3]);
        }
    }
}

// inclusive prefix over the lanes of a warp (also on two 16-bit halves at once, as long as no half overflows)
__device__ __forceinline__ uint32_t warp_inclusive(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, v, d);
        const uint32_t take = lane >= d ? 1u : 0u;   // loop invariant in every caller
        // one multiply-add per step.  (A predicated add would also be one instruction, but 16 interleaved scans would need 16
        // live predicates and the 7 predicate registers serialise them; written in C the compiler turns this into SEL + IADD.)
        asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(v) : "r"(o), "r"(take));
    }
    return v;
}
// 2^23 + x as a float for the low (HI = false) or high 16 bits of a packed register: one byte permute
template <bool HI>
__device__ __forceinline__ float magic16(uint32_t packed) {
    return __uint_as_float(__byte_perm(packed, 0x4B000000u, HI ? 0x7432 : 0x7410));
}

// exclusive prefix over the lanes of a warp
__device__ __forceinline__ int warp_exclusive(int v, int lane) {
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    return incl - v;
}

// ---- 2. checkpoints: S at row (j * BAND - radius - 2) for every band j >= 1 ------------------------------------------------
// The only sequential pass, so it carries nothing but the chain and has no block-level synchronisation:
//   Rgba: one WARP per (32-pixel window, channel pair {0,2} or {1,3}); lane = one pixel; the two channels ride in the 16-bit
//         halves of one register through a single warp scan (window sums <= 32 * 255);
//   gray: one warp per 32-unit window; lane = 4 pixels (4 chains), one scan of the lane totals.
// Rows are taken PF at a time: the loads of the next PF rows are in flight while the PF independent scans of the current ones
// run.  A short head makes every checkpoint row the last row of a PF-chunk.
template <int CH>
__global__ void __launch_bounds__(128) box_checkpoints(const BoxParams p) {
    constexpr int PF = 16;
    constexpr int NC = CH == 4 ? 2 : 4;   // chains per lane
    constexpr int WPW = CH == 4 ? 2 : 1;  // warps per window
    const int lane = threadIdx.x & 31;
    const int gw = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int win = gw / WPW;
    const int kp = gw % WPW;              // Rgba: channels kp and kp + 2
    if (win >= p.n_win) return;
    const int unit = win * 32 + lane;
    const bool in_row = unit < p.row_units;
    const bool full = CH == 4 || 4 * unit + 4 <= p.row_bytes;
    const uint8_t* colp = p.src + 4 * (size_t)unit;
    const float2* offp = reinterpret_cast<const float2*>(p.offs32) + 2 * win + kp;   // gray: .x only (kp == 0)
    float S[NC];
#pragma unroll
    for (int i = 0; i < NC; ++i) S[i] = 0.0f;
    const int y_end = (p.n_bands - 1) * BAND - p.radius - 2;   // last checkpoint row (< rows)

    uint32_t un[PF];
    float2 offn[PF];
    const size_t off_pitch = 2 * (size_t)p.n_win;
    auto fetch = [&](int y0) {   // rows y0 .. y0 + PF - 1, all <= y_end: every chunk ends on or before the last checkpoint row
        const uint8_t* q = colp + (size_t)y0 * p.src_pitch;
        const float2* o = offp + (size_t)y0 * off_pitch;
#pragma unroll
        for (int i = 0; i < PF; ++i) {
            uint32_t v = 0;
            if (in_row) {
                if (full) v = __ldg(reinterpret_cast<const uint32_t*>(q));
                else for (int b = 0; 4 * unit + b < p.row_bytes; ++b) v |= (uint32_t)q[b] << (8 * b);
            }
            un[i] = v;
            offn[i] = __ldg(o);
            q += p.src_pitch;
            o += off_pitch;
        }
    };
    // rows [y0, y0 + n) with the loads already in un / offn; the next chunk's loads are issued first
    auto chunk = [&](int y0, int n, int y_next) {
        uint32_t u[PF];
        float2 off[PF];
#pragma unroll
        for (int i = 0; i < PF; ++i) { u[i] = un[i]; off[i] = offn[i]; }
        if (y_next <= y_end) fetch(y_next);
        float pv[PF][NC];
#pragma unroll
        for (int i = 0; i < PF; ++i) {   // PF independent scans
            if constexpr (CH == 4) {
                const uint32_t incl = warp_inclusive(__byte_perm(u[i], 0, kp ? 0x4341 : 0x4240), lane);   // channel kp | channel kp+2 << 16
                pv[i][0] = __fadd_rn(magic16<false>(incl), off[i].x);
                pv[i][1] = __fadd_rn(magic16<true>(incl), off[i].y);
            } else {
                // 4 pixels of the lane: inclusive local prefix in two packed registers (p0 | p0+p1 << 16, .. + p2 | .. + p3 << 16)
                const uint32_t b0 = u[i] & 0xFFu, b1 = (u[i] >> 8) & 0xFFu, b2 = (u[i] >> 16) & 0xFFu, b3 = u[i] >> 24;
                const uint32_t tot = b0 + b1 + b2 + b3;
                const uint32_t excl = warp_inclusive(tot, lane) - tot;      // < 32 * 1020
                const uint32_t l01 = (excl + b0) | ((excl + b0 + b1) << 16);
                const uint32_t l23 = (excl + b0 + b1 + b2) | ((excl + tot) << 16);
                pv[i][0] = __fadd_rn(magic16<false>(l01), off[i].x);
                pv[i][1] = __fadd_rn(magic16<true>(l01), off[i].x);
                pv[i][2] = __fadd_rn(magic16<false>(l23), off[i].x);
                pv[i][3] = __fadd_rn(magic16<true>(l23), off[i].x);
            }
        }
#pragma unroll
        for (int i = 0; i < PF; ++i)     // the chains, row by row
            if (i < n) {
#pragma unroll
                for (int c = 0; c < NC; ++c) S[c] = __fadd_rn(S[c], pv[i][c]);
            }
    };

    const int head = (BAND - p.radius - 1) % PF;   // rows before the PF-aligned part
    fetch(0);
    int y = 0;
    if (head > 0) {
        chunk(0, head, head);
        y = head;
    }
    for (int jb = 1; jb < p.n_bands; ++jb) {
        const int yq = jb * BAND - p.radius - 2;   // S of this row resumes band jb; (yq - y + 1) is a multiple of PF
        for (; y <= yq; y += PF) chunk(y, PF, y + PF);
        float* ck = p.ckpt + (size_t)jb * p.ck_pitch + (size_t)unit * 4;
        if constexpr (CH == 4) {
            ck[kp] = S[0];
            ck[kp + 2] = S[1];
        } else {
#pragma unroll
            for (int c = 0; c < 4; ++c) ck[c] = S[c];
        }
    }
}

// ---- 3. chains from the checkpoint, SAT ring, evaluation ---------------------------------------------------------------------
// meta.clamp(u8, fl(m / area)) [blur] or meta.clamp(u8, fl(2*orig - fl(m / area))) [sharpen] WITHOUT the exact division.
// m is an integer (a combination of integer-valued floats) and area <= 31*31, so the exact value v is either a tie k + 1/2
// -- which the reference's correctly rounded divide represents exactly and then rounds away from zero -- or at least
// 1/(2*961) = 5.2e-4 away from every tie, far more than the 3e-5 that q = m * RN(1/area) can be off for |q| <= 256 (larger |q|
// saturate either way).  Hence trunc(q + 1/2 + 1e-4) is the reference's result for q >= 0, and every negative value clamps to 0
// exactly as its round-half-away does.  The float -> u8 conversion saturates: one instruction truncates and clamps both sides.
__device__ __forceinline__ uint32_t round_clamp_u8(float q) {
    uint32_t r;
    asm("cvt.rzi.u8.f32 %0, %1;" : "=r"(r) : "f"(__fadd_rn(q, 0.5001f)));
    return r;
}

// MODE 1: box blur, MODE 2: sharpen, MODE 3: adaptive mean threshold (gray only) (grid = n_strips x n_bands).
// The threshold compares the source with fl(fl(S / area) - c) for an arbitrary f32 c, so the rounding argument above does not
// carry over: MODE 3 forms the correctly rounded quotient (binary.zig:110-113).
template <int CH, int MODE>
__global__ void __launch_bounds__(BF_THREADS) box_chain(const BoxParams p) {
    extern __shared__ float smem_f[];
    float* pt = smem_f;                 // [GR][SE]  P tile (swizzled)
    float* ring = smem_f + GR * SE;     // [ring][SE] SAT rows (MODE != 0)
    const int t = threadIdx.x, lane = t & 31, wrow = t >> 5;
    const int strip = blockIdx.x;
    const int band = blockIdx.y;
    const int unit0 = strip * p.ou - p.mu;           // first unit of the strip (may be negative)
    const int elem0 = unit0 * 4;
    const int y0 = band * BAND;
    const int y1 = min(p.rows, y0 + BAND);
    const int ys = max(0, y0 - p.radius - 1);         // first chain row
    const int y_last = y1 - 1 + p.radius;             // last (possibly virtual) chain row
    const int rmask = p.ring - 1;

    // chains: thread t owns element columns t and t + 256 of the strip
    float s0 = 0.0f, s1 = 0.0f;
    if (ys > 0) {   // resume from the checkpoint (columns outside the image are never read by an output)
        const float* ck = p.ckpt + (size_t)band * p.ck_pitch;
        const int e0 = elem0 + t, e1 = elem0 + t + 256;
        s0 = (e0 >= 0 && e0 < p.ck_pitch) ? ck[e0] : 0.0f;
        s1 = (e1 >= 0 && e1 < p.ck_pitch) ? ck[e1] : 0.0f;
    }

    // evaluation geometry of this thread's unit: loop invariant (the column window never changes)
    float* zrow = ring + p.ring * SE;                 // 16 zero floats: the SAT left of / above the image
    if (t < 16) zrow[t] = 0.0f;
    const int ev_unit = strip * p.ou + (t & (SU - 1));
    const bool ev_active = (t & (SU - 1)) < min(p.ou, p.row_units - strip * p.ou);
    constexpr int NJ = CH == 4 ? 1 : 4;               // distinct pixel columns per unit
    int ed[NJ], el[NJ], wcols[NJ];
    bool has_left[NJ];
    float area_full[NJ], rcp_full[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
        const int c = CH == 4 ? ev_unit : min(4 * ev_unit + j, p.cols - 1);
        const int c1 = max(c - p.radius, 0), c2 = min(c + p.radius, p.cols - 1);
        ed[j] = (CH == 4 ? 4 * c2 : c2) - elem0;              // local element of column c2 (channel 0)
        el[j] = (CH == 4 ? 4 * (c1 - 1) : c1 - 1) - elem0;    // local element of column c1 - 1
        has_left[j] = c1 > 0;
        wcols[j] = c2 - c1 + 1;
        area_full[j] = (float)((2 * p.radius + 1) * wcols[j]);
        rcp_full[j] = __frcp_rn(area_full[j]);
    }
    uint8_t* dcol = p.dst + 4 * (size_t)ev_unit;

    // the loads of a block are issued one block ahead of their use
    uint32_t un[4] = {0u, 0u, 0u, 0u};
    float4 offn = make_float4(0.f, 0.f, 0.f, 0.f);
    auto fetch = [&](int y) {
        if (y < p.rows) {
            const uint8_t* rowp = p.src + (size_t)y * p.src_pitch;
#pragma unroll
            for (int j = 0; j < 4; ++j) un[j] = load_unit<CH>(rowp, unit0 + 4 * lane + j, p.row_units, p.row_bytes);
            offn = __ldg(reinterpret_cast<const float4*>(p.offs + ((size_t)y * p.n_strips + strip) * 4));
        }
    };
    fetch(ys + wrow);

    for (int yb = ys; yb <= y_last; yb += GR) {
        // ---- P phase: warp `wrow` owns row yb + wrow; lane l owns units 4l .. 4l+3 of the strip.  All integer work rides in
        // 16-bit halves (in-strip prefixes are <= 512 * 255 / 4 .. < 2^16); P = (2^23 + in-strip prefix) + (strip offset - 2^23).
        {
            const int y = yb + wrow;
            const uint32_t u[4] = {un[0], un[1], un[2], un[3]};
            const float4 off = offn;
            if (yb + GR <= y_last) fetch(y + GR);
            // (rows past the image end compute on stale registers; the chain phase never reads their tile row)
            float* dstp = pt + wrow * SE;
            if constexpr (CH == 4) {
                uint32_t l02[4], l13[4];   // inclusive local prefix: channels {0,2} and {1,3} in 16-bit halves
                l02[0] = __byte_perm(u[0], 0, 0x4240);
                l13[0] = __byte_perm(u[0], 0, 0x4341);
#pragma unroll
                for (int j = 1; j < 4; ++j) {
                    l02[j] = l02[j - 1] + __byte_perm(u[j], 0, 0x4240);
                    l13[j] = l13[j - 1] + __byte_perm(u[j], 0, 0x4341);
                }
                const uint32_t e02 = warp_inclusive(l02[3], lane) - l02[3];   // exclusive over lanes: <= 124 * 255 per half
                const uint32_t e13 = warp_inclusive(l13[3], lane) - l13[3];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t a = e02 + l02[j], b = e13 + l13[j];
                    float4 f;
                    f.x = __fadd_rn(magic16<false>(a), off.x);
                    f.y = __fadd_rn(magic16<false>(b), off.y);
                    f.z = __fadd_rn(magic16<true>(a), off.z);
                    f.w = __fadd_rn(magic16<true>(b), off.w);
                    *reinterpret_cast<float4*>(dstp + pt_chunk(4 * lane + j) * 4) = f;
                }
            } else {
                uint32_t tot[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) tot[j] = __dp4a(u[j], 0x01010101u, 0u);
                const uint32_t lane_tot = tot[0] + tot[1] + tot[2] + tot[3];
                uint32_t run = warp_inclusive(lane_tot, lane) - lane_tot;     // < 512 * 255 = 130560: needs 17 bits, so no packing here
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t b0 = u[j] & 0xFFu, b1 = (u[j] >> 8) & 0xFFu, b2 = (u[j] >> 16) & 0xFFu;
                    float4 f;
                    f.x = __fadd_rn(__uint_as_float(0x4B000000u | (run + b0)), off.x);
                    f.y = __fadd_rn(__uint_as_float(0x4B000000u | (run + b0 + b1)), off.x);
                    f.z = __fadd_rn(__uint_as_float(0x4B000000u | (run + b0 + b1 + b2)), off.x);
                    run += tot[j];
                    f.w = __fadd_rn(__uint_as_float(0x4B000000u | run), off.x);
                    *reinterpret_cast<float4*>(dstp + pt_chunk(4 * lane + j) * 4) = f;
                }
            }
        }
        __syncthreads();
        // ---- chain phase
        {
            const int i0 = pt_index(t), i1 = pt_index(t + 256);
#pragma unroll
            for (int g = 0; g < GR; ++g) {
                const int y = yb + g;
                if (y < p.rows) {
                    s0 = __fadd_rn(s0, pt[g * SE + i0]);
                    s1 = __fadd_rn(s1, pt[g * SE + i1]);
                    float* rr = ring + (y & rmask) * SE;
                    rr[t] = s0;
                    rr[t + 256] = s1;
                }
            }
        }
        __syncthreads();
        // ---- evaluation of the output rows this block completed: yo = y - radius (thread: one unit, rows g, g+2, ..)
        if (ev_active) {
            for (int g = t >> 7; g < GR; g += BF_THREADS / SU) {
                const int yo = yb + g - p.radius;
                if (yo < y0 || yo >= y1) continue;
                const int r1 = max(yo - p.radius, 0), r2 = min(yo + p.radius, p.rows - 1);
                const int h = r2 - r1 + 1;
                const float* row_d = ring + (r2 & rmask) * SE;
                const float* row_t = r1 > 0 ? ring + ((r1 - 1) & rmask) * SE : zrow;   // above the image: zeros
                uint32_t orig = 0;
                if constexpr (MODE >= 2) orig = load_unit<CH>(p.src + (size_t)yo * p.src_pitch, ev_unit, p.row_units, p.row_bytes);
                uint32_t packed = 0;
                if constexpr (CH == 4) {
                    float area = area_full[0], rcp = rcp_full[0];
                    if (h != 2 * p.radius + 1) {
                        area = (float)(h * wcols[0]);
                        rcp = __frcp_rn(area);
                    }
                    const float4 D = *reinterpret_cast<const float4*>(row_d + ed[0]);
                    const float4 T = *reinterpret_cast<const float4*>(row_t + (r1 > 0 ? ed[0] : 0));
                    const float4 Lf = *reinterpret_cast<const float4*>(has_left[0] ? row_d + el[0] : zrow);
                    const float4 Cn = *reinterpret_cast<const float4*>((has_left[0] && r1 > 0) ? row_t + el[0] : zrow);
                    const float dv[4] = {D.x, D.y, D.z, D.w}, lv[4] = {Lf.x, Lf.y, Lf.z, Lf.w};
                    const float tv[4] = {T.x, T.y, T.z, T.w}, cv[4] = {Cn.x, Cn.y, Cn.z, Cn.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float sum = __fadd_rn(__fsub_rn(__fsub_rn(dv[j], lv[j]), tv[j]), cv[j]);   // integral.zig:86-89
                        float val = __fmul_rn(sum, rcp);
                        if constexpr (MODE == 2) val = __fsub_rn((float)(2u * ((orig >> (8 * j)) & 0xFFu)), val);   // integral.zig:357 (2 * orig is exact)
                        packed |= round_clamp_u8(val) << (8 * j);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (4 * ev_unit + j >= p.cols) break;
                        float area = area_full[j], rcp = rcp_full[j];
                        if (h != 2 * p.radius + 1) {
                            area = (float)(h * wcols[j]);
                            rcp = __frcp_rn(area);
                        }
                        const float D = row_d[ed[j]];
                        const float top = row_t[r1 > 0 ? ed[j] : 0];
                        const float left = has_left[j] ? row_d[el[j]] : 0.0f;
                        const float corner = (has_left[j] && r1 > 0) ? row_t[el[j]] : 0.0f;
                        const float sum = __fadd_rn(__fsub_rn(__fsub_rn(D, left), top), corner);
                        if constexpr (MODE == 3) {
                            const float thr = __fsub_rn(__fdiv_rn(sum, area), p.c);   // mean - c
                            packed |= ((float)((orig >> (8 * j)) & 0xFFu) > thr ? 255u : 0u) << (8 * j);
                            continue;
                        }
                        float val = __fmul_rn(sum, rcp);
                        if constexpr (MODE == 2) val = __fsub_rn((float)(2u * ((orig >> (8 * j)) & 0xFFu)), val);
                        packed |= round_clamp_u8(val) << (8 * j);
                    }
                }
                uint8_t* dpx = dcol + (size_t)yo * p.dst_pitch;
                if (CH == 4 || 4 * ev_unit + 4 <= p.row_bytes) {
                    *reinterpret_cast<uint32_t*>(dpx) = packed;
                } else {
                    for (int b = 0; 4 * ev_unit + b < p.row_bytes; ++b) dpx[b] = (uint8_t)(packed >> (8 * b));
                }
            }
            // no barrier needed here: a thread only reaches the next chain phase (the next ring write) through the barrier after
            // the next P phase, which every thread enters after finishing this loop
        }
    }
}

template <int CH>
int launch_all(const BoxParams& p, int mode, float* offs, float* offs32, cudaStream_t s) {
    box_row_offsets<CH><<<div_up(p.rows, 8), 256, 0, s>>>(p, offs, offs32);
    ZB_LAUNCHED();
    const int smem_ev = ((GR + p.ring) * SE + 16) * (int)sizeof(float);
    if (p.n_bands > 1) {
        const int warps = CH == 4 ? 2 * p.n_win : p.n_win;
        box_checkpoints<CH><<<div_up(warps, 4), 128, 0, s>>>(p);
        ZB_LAUNCHED();
    }
    dim3 grid(p.n_strips, p.n_bands);
    if (mode == 3) {
        if constexpr (CH == 1) {
            ZB_CUDA(cudaFuncSetAttribute(box_chain<CH, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_ev));
            box_chain<CH, 3><<<grid, BF_THREADS, smem_ev, s>>>(p);
        } else {
            return ZB_ERR_UNSUPPORTED;
        }
    } else if (mode == 2) {
        ZB_CUDA(cudaFuncSetAttribute(box_chain<CH, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_ev));
        box_chain<CH, 2><<<grid, BF_THREADS, smem_ev, s>>>(p);
    } else {
        ZB_CUDA(cudaFuncSetAttribute(box_chain<CH, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_ev));
        box_chain<CH, 1><<<grid, BF_THREADS, smem_ev, s>>>(p);
    }
    ZB_LAUNCHED();
    return ZB_OK;
}

}  // namespace

// Returns ZB_ERR_UNSUPPORTED outside the fused envelope (the caller then builds the SAT in HBM).
// mode: 1 box blur, 2 sharpen, 3 adaptive mean threshold (gray; c is subtracted from the mean).
int box_fused_u8(const zb_image* src, zb_image* dst, int channels, uint32_t radius, int mode, float c, cudaStream_t s) {
    if (channels != 1 && channels != 4) return ZB_ERR_UNSUPPORTED;
    if (mode == 3 && channels != 1) return ZB_ERR_UNSUPPORTED;
    if (radius == 0 || radius > 15) return ZB_ERR_UNSUPPORTED;                 // ring <= 64 rows (128 KB), margins <= 16 units
    if (images_overlap(src, dst, (size_t)channels)) return ZB_ERR_UNSUPPORTED;  // bands would race with in-place / overlapping rows
    if ((uint64_t)src->cols * 255u >= (1u << 24)) return ZB_ERR_UNSUPPORTED;   // row prefixes must be exact in f32
    if (src->rows > (1u << 30) || src->cols > (1u << 28)) return ZB_ERR_UNSUPPORTED;
    const size_t sp = (size_t)src->stride * channels, dp = (size_t)dst->stride * channels;
    if (((uintptr_t)src->data & 3u) || ((uintptr_t)dst->data & 3u) || (sp & 3u) || (dp & 3u)) return ZB_ERR_UNSUPPORTED;
    BoxParams p;
    p.src = (const uint8_t*)src->data;
    p.dst = (uint8_t*)dst->data;
    p.src_pitch = sp;
    p.dst_pitch = dp;
    p.rows = (int)src->rows;
    p.cols = (int)src->cols;
    p.row_bytes = p.cols * channels;
    p.row_units = (p.row_bytes + 3) / 4;
    p.radius = (int)radius;
    p.c = c;
    p.mu = channels == 4 ? p.radius + 1 : (p.radius + 1 + 3) / 4;
    p.ou = SU - 2 * p.mu;
    p.n_strips = (p.row_units + p.ou - 1) / p.ou;
    p.n_bands = (p.rows + BAND - 1) / BAND;
    int ring = 16;
    while (ring < 2 * p.radius + 2 + GR) ring <<= 1;
    p.ring = ring;
    p.n_win = (p.row_units + 31) / 32;
    p.ck_pitch = p.n_win * 128;
    Scratch offs, offs32, ckpt;
    int rc = offs.alloc((size_t)p.rows * p.n_strips * 4 * sizeof(int), s);
    if (rc) return rc;
    if ((rc = offs32.alloc((size_t)p.rows * p.n_win * 4 * sizeof(int), s))) return rc;
    if ((rc = ckpt.alloc((size_t)p.n_bands * p.ck_pitch * sizeof(float), s))) return rc;
    p.offs = offs.as<float>();
    p.offs32 = offs32.as<float>();
    p.ckpt = ckpt.as<float>();
    t_last_kernel = mode == 3 ? "box_fused_threshold" : (mode == 2 ? "box_fused_sharpen" : "box_fused_blur");
    return channels == 4 ? launch_all<4>(p, mode, offs.as<float>(), offs32.as<float>(), s)
                         : launch_all<1>(p, mode, offs.as<float>(), offs32.as<float>(), s);
}

}  // namespace zb
