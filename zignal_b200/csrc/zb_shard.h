// zb_shard.h -- internals of the multi-GPU layer (zb_shard.cu) shared with the kernels that take part in it
// (zb_conv_fused.cu: halo rows read from the row neighbours' memory inside the convolution kernel; zb_fdm.cu: the
// 11-moment all-gather inside the statistics kernel).
//
// One process per GPU.  Every rank owns a small CONTROL BLOCK in device memory that all other ranks map through CUDA IPC;
// neighbours signal each other with system-scope release stores into it and poll their own copy with acquire loads:
//   ready_from[d]  "the source of sharded op #e is complete on the neighbour in direction d" (0 = up, 1 = down)
//   done_from[d]   "the neighbour in direction d has finished reading my edge rows for op #e"
//   gather[e&1][r] the payload rank r contributed to the small all-gather of op #e (word 15 = e, written last)
// Op numbers (`epoch`) are a host-side counter every rank advances identically (SPMD call order).
#pragma once
#include "zb_internal.h"

#define ZB_SHARD_MAX_WORLD 16

namespace zb {

struct ShardCtrl {
    unsigned long long ready_from[2];
    unsigned long long done_from[2];
    unsigned long long gather[2][ZB_SHARD_MAX_WORLD][16];
    unsigned long long halo_landed;   // local: op number whose neighbour rows have all arrived in my halo rows
    unsigned int halo_reads[2];   // local: [0] CTAs of the running kernel whose share of the halo copy is done
    unsigned int exit_ticket;     // local: CTAs that have left the running kernel
    unsigned int error;           // local: set when a wait timed out (a peer never arrived)
    unsigned int gather_ticket;   // local: blocks of the running statistics kernel that have added their partial sums
    unsigned int pad[3];
};

// What a kernel needs to talk to its row neighbours.  All pointers are in THIS process's address space (peer pointers are
// IPC mappings).  A null `up` / `down` control pointer means "no neighbour on that side" (global image edge).
struct ShardLink {
    ShardCtrl* self;
    ShardCtrl* up;
    ShardCtrl* down;
    unsigned long long epoch;
};

// all ranks' control blocks, for the one-shot all-gather
struct ShardAll {
    ShardCtrl* ctrl[ZB_SHARD_MAX_WORLD];
    int rank, world;
    unsigned long long epoch;
};

#ifdef __CUDACC__
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// Spin until *flag >= epoch.  A peer that never arrives (crashed rank, mismatched call order) must not hang the GPU:
// after ~20 s the wait gives up and records the failure in the control block (zb_shard_status reports it).
static __device__ __forceinline__ bool shard_wait_ge(const unsigned long long* flag, unsigned long long epoch, ShardCtrl* self) {
    if (ld_acquire_sys(flag) >= epoch) return true;
    const unsigned long long t0 = global_timer_ns();
    unsigned spins = 0;
    while (ld_acquire_sys(flag) < epoch) {
        if ((++spins & 1023u) == 0 && global_timer_ns() - t0 > 20000000000ull) {
            atomicExch(&self->error, 1u);
            return false;
        }
    }
    return true;
}
#endif

}  // namespace zb

// ---- host side ---------------------------------------------------------------------------------------------------
struct zb_shard_alloc_rec {
    void* base = nullptr;
    size_t bytes = 0;
    void* peer[ZB_SHARD_MAX_WORLD] = {};   // this allocation in every rank's ... mapped into this process (self = base)
};

struct zb_shard_comm;
struct zb_shard_image {
    zb_shard_comm* comm;
    int pixfmt;
    uint32_t cols;
    uint32_t halo_cap;                      // rows of padding this rank owns above and below its block
    uint32_t rows[ZB_SHARD_MAX_WORLD];      // block heights, rank order
    uint64_t stride[ZB_SHARD_MAX_WORLD];    // in pixels
    void* data[ZB_SHARD_MAX_WORLD];         // interior row 0 of every rank's block (peer mappings; null without peer access)
};

namespace zb {
// accessors used by other translation units
int shard_link(zb_shard_comm* c, int border, bool advance_epoch, ShardLink* out, int* up_rank, int* down_rank);
int shard_all(zb_shard_comm* c, bool advance_epoch, ShardAll* out);
bool shard_peer_ok(const zb_shard_comm* c);
int shard_world(const zb_shard_comm* c);
int shard_rank(const zb_shard_comm* c);
// in-place sum over all ranks through NCCL (dtype: 0 = f32, 1 = f64, 2 = u64)
int shard_allreduce(zb_shard_comm* c, void* buf, size_t count, int dtype, cudaStream_t s);

// zb_conv_fused.cu: the fused RGBA f32 convolution of a row block whose edge rows come from the neighbours' memory
// (copied over NVLink into the block's halo rows by the kernel's own prologue).  up / down: block geometry of the neighbours (null data = global edge).
struct PeerBlock {
    const void* data;   // row 0 of the neighbour's block
    uint32_t rows;
    uint64_t stride;
};
int conv_separable_fused_rgbaf32_shard(const zb_image* src, zb_image* dst, const float* kx, int nx, const float* ky, int ny, int border,
                                       bool exact, const PeerBlock& up, const PeerBlock& down, uint32_t halo_cap, const ShardLink& link,
                                       cudaStream_t s);
}  // namespace zb
