// zb_shard.cu -- the multi-GPU layer behind the C ABI (SURVEY.md 8(e)): one process per GPU, a large image sharded into
// row blocks, a batch split into contiguous shares, statistics combined across ranks.
//
// The reference is single-process (no counterpart file); the partitioning follows SURVEY 8(e):
//   convolution / blur   row blocks, the `half` edge rows of the row neighbours are the only data that crosses GPUs
//   box blur, sharpen, dense convolve, order statistics, ...   same, through zb_shard_halo_exchange + the ordinary entry point
//   resize / rotate / warp batches   zb_shard_split, no exchange
//   fdm                  11 integer moments all-gathered over peer memory inside the statistics kernel (zb_fdm.cu)
//   pca                  one NCCL all-reduce of the dim x dim partial products (zb_shard_allreduce)
//
// Plumbing: NCCL (dlopen'ed, the torch-bundled libnccl.so.2 or the system one) bootstraps the communicator, exchanges the
// CUDA IPC handles and serves as the fallback exchange; the data path proper uses IPC peer mappings over NVLink -- the fused
// convolution kernel TMA-loads the neighbours' rows itself (zb_conv_fused.cu), the halo exchange of every other filter is one
// pull kernel.  Synchronisation is a pair of flags per neighbour in a control block (zb_shard.h).
#include <dlfcn.h>

#include <mutex>
#include <string>
#include <vector>

#include "zb_conv.h"
#include "zb_shard.h"

namespace {

// ---- NCCL, resolved at run time (no link-time dependency; nothing is loaded unless a communicator is created) ----
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { kNcclUint8 = 1, kNcclUint64 = 5, kNcclFloat32 = 7, kNcclFloat64 = 8, kNcclSum = 0 };

struct NcclApi {
    void* handle = nullptr;
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int*) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

int nccl_fail(int r, const char* what) {
    snprintf(zb::t_last_error, sizeof(zb::t_last_error), "NCCL %s: %s", what, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    return ZB_ERR_DEVICE_FAILURE;
}
#define ZB_NCCL(expr)                                  \
    do {                                               \
        int _r = (expr);                               \
        if (_r != 0) return nccl_fail(_r, #expr);      \
    } while (0)

int load_nccl() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.handle) return ZB_OK;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);   // already in the process (torch loads its own copy)
    if (!h) {
        // the copy next to torch (same directory layout as the interpreter that loaded us), then the system one
        Dl_info info;
        std::vector<std::string> candidates;
        if (const char* env = getenv("ZB_NCCL_LIB")) candidates.push_back(env);
        if (dladdr((void*)&load_nccl, &info) && info.dli_fname) {
            std::string p(info.dli_fname);   // .../zignal_b200/lib/libzignal_b200.so
            (void)p;
        }
        candidates.push_back("/opt/prime-rl/.venv/lib/python3.12/site-packages/nvidia/nccl/lib/libnccl.so.2");
        candidates.push_back("libnccl.so.2");
        candidates.push_back("libnccl.so");
        for (const std::string& c : candidates) {
            h = dlopen(c.c_str(), RTLD_NOW | RTLD_GLOBAL);
            if (h) break;
        }
    }
    if (!h) {
        snprintf(zb::t_last_error, sizeof(zb::t_last_error), "libnccl.so.2 not found (set ZB_NCCL_LIB): %s", dlerror());
        return ZB_ERR_DEVICE_FAILURE;
    }
    NcclApi a;
    a.handle = h;
#define ZB_SYM(field, name)                                                                   \
    *(void**)(&a.field) = dlsym(h, name);                                                     \
    if (!a.field) {                                                                           \
        snprintf(zb::t_last_error, sizeof(zb::t_last_error), "libnccl: missing symbol %s", name); \
        return ZB_ERR_DEVICE_FAILURE;                                                         \
    }
    ZB_SYM(GetUniqueId, "ncclGetUniqueId")
    ZB_SYM(CommInitRank, "ncclCommInitRank")
    ZB_SYM(CommDestroy, "ncclCommDestroy")
    ZB_SYM(AllGather, "ncclAllGather")
    ZB_SYM(AllReduce, "ncclAllReduce")
    ZB_SYM(Send, "ncclSend")
    ZB_SYM(Recv, "ncclRecv")
    ZB_SYM(GroupStart, "ncclGroupStart")
    ZB_SYM(GroupEnd, "ncclGroupEnd")
    ZB_SYM(GetErrorString, "ncclGetErrorString")
    ZB_SYM(GetVersion, "ncclGetVersion")
#undef ZB_SYM
    g_nccl = a;
    return ZB_OK;
}

std::atomic<int> g_shard_path{0};   // 0 auto, 1 force the NCCL send/recv exchange, 2 force the peer pull kernel (no fused peer loads)

}  // namespace

struct zb_shard_comm {
    int rank = 0, world = 1, device = 0;
    ncclComm_t nccl = nullptr;
    bool peer_ok = false;
    zb::ShardCtrl* ctrl[ZB_SHARD_MAX_WORLD] = {};   // every rank's control block (self = the local allocation)
    unsigned long long epoch = 0;
    std::vector<zb_shard_alloc_rec> allocs;
    void* staging = nullptr;   // device scratch for the bootstrap all-gathers (4 KB per rank)
    cudaStream_t boot = nullptr;
};

namespace {

using namespace zb;

// all-gather `bytes` (<= 4096) of host data from every rank into out[world][bytes]
int gather_host(zb_shard_comm* c, const void* mine, size_t bytes, void* out) {
    if (bytes > 4096) return ZB_ERR_INVALID_ARGUMENT;
    if (c->world == 1) { memcpy(out, mine, bytes); return ZB_OK; }
    char* st = (char*)c->staging;                         // [0, 4096): send, [4096, ...): recv
    ZB_CUDA(cudaMemcpyAsync(st, mine, bytes, cudaMemcpyHostToDevice, c->boot));
    ZB_NCCL(g_nccl.AllGather(st, st + 4096, bytes, kNcclUint8, c->nccl, c->boot));
    ZB_CUDA(cudaMemcpyAsync(out, st + 4096, bytes * c->world, cudaMemcpyDeviceToHost, c->boot));
    ZB_CUDA(cudaStreamSynchronize(c->boot));
    return ZB_OK;
}

// Map `local` (a cudaMalloc allocation of this rank) into every other rank.  peers[r] receives rank r's allocation as seen from
// here.  Returns ZB_ERR_UNSUPPORTED (and leaves peers untouched) if any rank could not export or import a handle.
int exchange_ipc(zb_shard_comm* c, void* local, void** peers) {
    struct Msg { cudaIpcMemHandle_t h; int ok; int device; };
    Msg mine;
    memset(&mine, 0, sizeof(mine));
    mine.ok = cudaIpcGetMemHandle(&mine.h, local) == cudaSuccess ? 1 : 0;
    if (!mine.ok) cudaGetLastError();
    mine.device = c->device;
    std::vector<Msg> all(c->world);
    int rc = gather_host(c, &mine, sizeof(Msg), all.data());
    if (rc) return rc;
    int ok = 1;
    for (int r = 0; r < c->world; ++r) ok &= all[r].ok;
    std::vector<void*> mapped(c->world, nullptr);
    if (ok) {
        for (int r = 0; r < c->world && ok; ++r) {
            if (r == c->rank) { mapped[r] = local; continue; }
            void* p = nullptr;
            if (cudaIpcOpenMemHandle(&p, all[r].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                snprintf(t_last_error, sizeof(t_last_error), "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(cudaGetLastError()));
                ok = 0;
            } else {
                mapped[r] = p;
            }
        }
    }
    // every rank must agree, or the ranks would take different paths
    int agree[ZB_SHARD_MAX_WORLD];
    if ((rc = gather_host(c, &ok, sizeof(int), agree))) return rc;
    int all_ok = 1;
    for (int r = 0; r < c->world; ++r) all_ok &= agree[r];
    if (!all_ok) {
        for (int r = 0; r < c->world; ++r)
            if (r != c->rank && mapped[r]) cudaIpcCloseMemHandle(mapped[r]);
        return ZB_ERR_UNSUPPORTED;
    }
    for (int r = 0; r < c->world; ++r) peers[r] = mapped[r];
    return ZB_OK;
}

const zb_shard_alloc_rec* find_alloc(const zb_shard_comm* c, const void* p, int* index) {
    for (size_t i = 0; i < c->allocs.size(); ++i) {
        const char* b = (const char*)c->allocs[i].base;
        if (b && (const char*)p >= b && (const char*)p < b + c->allocs[i].bytes) {
            if (index) *index = (int)i;
            return &c->allocs[i];
        }
    }
    return nullptr;
}

// ---- the pull kernel: copy the neighbours' edge rows into this block's halo rows over NVLink ----------------------
struct PullParams {
    ShardLink link;
    const char* up_rows_src;     // first of the `reach` rows to fetch from the upper neighbour (its last rows), or null
    const char* down_rows_src;   // the lower neighbour's first rows, or null
    char* top_halo;              // local destination of the upper rows (row -reach of the block)
    char* bottom_halo;           // local destination (row `rows` of the block)
    unsigned long long src_up_pitch, src_down_pitch, dst_pitch;   // bytes
    unsigned long long row_bytes;
    int reach;
};

__global__ void __launch_bounds__(256) halo_pull_kernel(const PullParams p) {
    ShardCtrl* me = p.link.self;
    if (threadIdx.x == 0) {
        if (blockIdx.x == 0) {   // stream order: my block is complete
            if (p.link.up) st_release_sys(&p.link.up->ready_from[1], p.link.epoch);
            if (p.link.down) st_release_sys(&p.link.down->ready_from[0], p.link.epoch);
        }
        if (p.up_rows_src) shard_wait_ge(&me->ready_from[0], p.link.epoch, me);
        if (p.down_rows_src) shard_wait_ge(&me->ready_from[1], p.link.epoch, me);
    }
    __syncthreads();
    const bool vec = ((p.row_bytes | p.src_up_pitch | p.src_down_pitch | p.dst_pitch | (uintptr_t)p.up_rows_src | (uintptr_t)p.down_rows_src |
                       (uintptr_t)p.top_halo | (uintptr_t)p.bottom_halo) & 15u) == 0;
    for (int side = 0; side < 2; ++side) {
        const char* src = side == 0 ? p.up_rows_src : p.down_rows_src;
        if (!src) continue;
        char* dst = side == 0 ? p.top_halo : p.bottom_halo;
        const unsigned long long sp = side == 0 ? p.src_up_pitch : p.src_down_pitch;
        if (vec) {
            const unsigned long long per_row = p.row_bytes / 16, total = per_row * p.reach;
            for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (unsigned long long)gridDim.x * blockDim.x) {
                const unsigned long long r = i / per_row, e = i - r * per_row;
                const int4 v = *reinterpret_cast<const int4*>(src + r * sp + e * 16);
                *reinterpret_cast<int4*>(dst + r * p.dst_pitch + e * 16) = v;
            }
        } else {
            const unsigned long long total = p.row_bytes * p.reach;
            for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (unsigned long long)gridDim.x * blockDim.x) {
                const unsigned long long r = i / p.row_bytes, e = i - r * p.row_bytes;
                dst[r * p.dst_pitch + e] = src[r * sp + e];
            }
        }
    }
    // last block out: tell the neighbours their rows have been read, then wait until they have read mine
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&me->exit_ticket, 1u) == gridDim.x - 1u) {
            me->exit_ticket = 0;
            if (p.up_rows_src) st_release_sys(&p.link.up->done_from[1], p.link.epoch);
            if (p.down_rows_src) st_release_sys(&p.link.down->done_from[0], p.link.epoch);
            if (p.link.up) shard_wait_ge(&me->done_from[0], p.link.epoch, me);
            if (p.link.down) shard_wait_ge(&me->done_from[1], p.link.epoch, me);
        }
    }
}

void neighbours(const zb_shard_comm* c, int border, int* up, int* down) {
    const bool wrap = border == ZB_BORDER_WRAP;
    *up = c->rank > 0 ? c->rank - 1 : (wrap && c->world > 1 ? c->world - 1 : -1);
    *down = c->rank < c->world - 1 ? c->rank + 1 : (wrap && c->world > 1 ? 0 : -1);
}

}  // namespace

namespace zb {

bool shard_peer_ok(const zb_shard_comm* c) { return c && c->peer_ok; }
int shard_world(const zb_shard_comm* c) { return c ? c->world : 1; }
int shard_rank(const zb_shard_comm* c) { return c ? c->rank : 0; }

int shard_link(zb_shard_comm* c, int border, bool advance_epoch, ShardLink* out, int* up_rank, int* down_rank) {
    int up, down;
    neighbours(c, border, &up, &down);
    if (advance_epoch) ++c->epoch;
    out->self = c->ctrl[c->rank];
    out->up = up >= 0 ? c->ctrl[up] : nullptr;
    out->down = down >= 0 ? c->ctrl[down] : nullptr;
    out->epoch = c->epoch;
    if (up_rank) *up_rank = up;
    if (down_rank) *down_rank = down;
    return ZB_OK;
}

int shard_all(zb_shard_comm* c, bool advance_epoch, ShardAll* out) {
    if (advance_epoch) ++c->epoch;
    memset(out, 0, sizeof(*out));
    for (int r = 0; r < c->world; ++r) out->ctrl[r] = c->ctrl[r];
    out->rank = c->rank;
    out->world = c->world;
    out->epoch = c->epoch;
    return ZB_OK;
}

int shard_allreduce(zb_shard_comm* c, void* buf, size_t count, int dtype, cudaStream_t s) {
    if (!c || !buf) return ZB_ERR_INVALID_ARGUMENT;
    if (c->world == 1 || count == 0) return ZB_OK;
    const int dt = dtype == 0 ? kNcclFloat32 : (dtype == 1 ? kNcclFloat64 : (dtype == 2 ? kNcclUint64 : -1));
    if (dt < 0) return ZB_ERR_INVALID_ARGUMENT;
    ZB_NCCL(g_nccl.AllReduce(buf, buf, count, dt, kNcclSum, c->nccl, s));
    return ZB_OK;
}

}  // namespace zb

using namespace zb;

// halo rows of `img` on the two neighbour sides for a filter of vertical reach `reach` (pure host arithmetic)
static int view_of(const zb_shard_image* img, uint32_t reach, int border, zb_image* view, uint32_t* interior_first) {
    const zb_shard_comm* c = img->comm;
    int up, down;
    neighbours(c, border, &up, &down);
    const uint32_t rows = img->rows[c->rank];
    const uint64_t stride = img->stride[c->rank];
    const size_t pb = pixel_bytes(img->pixfmt);
    const uint32_t top = up >= 0 ? reach : 0, bottom = down >= 0 ? reach : 0;
    if (reach > img->halo_cap && (top || bottom)) return ZB_ERR_INVALID_ARGUMENT;
    view->data = (char*)img->data[c->rank] - (size_t)top * stride * pb;
    view->rows = rows + top + bottom;
    view->cols = img->cols;
    view->stride = stride;
    if (interior_first) *interior_first = top;
    return ZB_OK;
}

extern "C" {

int zb_shard_unique_id(uint8_t* id128) {
    if (!id128) return ZB_ERR_INVALID_ARGUMENT;
    int rc = load_nccl();
    if (rc) return rc;
    ncclUniqueId id;
    ZB_NCCL(g_nccl.GetUniqueId(&id));
    memcpy(id128, &id, 128);
    return ZB_OK;
}

int zb_shard_comm_create(zb_shard_comm** out, int rank, int world, const uint8_t* id128) {
    if (!out || world < 1 || world > ZB_SHARD_MAX_WORLD || rank < 0 || rank >= world) return ZB_ERR_INVALID_ARGUMENT;
    if (world > 1 && !id128) return ZB_ERR_INVALID_ARGUMENT;
    zb_shard_comm* c = new zb_shard_comm();
    c->rank = rank;
    c->world = world;
    auto fail = [&](int rc) { zb_shard_comm_destroy(c); return rc; };
    if (cudaGetDevice(&c->device) != cudaSuccess) return fail(ZB_ERR_DEVICE_FAILURE);
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return fail(rc);
    ShardCtrl* mine = nullptr;
    if (cudaMalloc(&mine, sizeof(ShardCtrl)) != cudaSuccess || cudaMemset(mine, 0, sizeof(ShardCtrl)) != cudaSuccess) return fail(ZB_ERR_OUT_OF_MEMORY);
    c->ctrl[rank] = mine;
    if (world == 1) { *out = c; return ZB_OK; }
    if ((rc = load_nccl())) return fail(rc);
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    { int r = g_nccl.CommInitRank(&c->nccl, world, id, rank); if (r) return fail(nccl_fail(r, "ncclCommInitRank")); }
    if (cudaStreamCreateWithFlags(&c->boot, cudaStreamNonBlocking) != cudaSuccess) return fail(ZB_ERR_DEVICE_FAILURE);
    if (cudaMalloc(&c->staging, 4096 * (size_t)(world + 1)) != cudaSuccess) return fail(ZB_ERR_OUT_OF_MEMORY);
    if (cudaDeviceSynchronize() != cudaSuccess) return fail(ZB_ERR_DEVICE_FAILURE);   // the memset above precedes any peer's first store
    void* peers[ZB_SHARD_MAX_WORLD] = {};
    rc = exchange_ipc(c, mine, peers);
    if (rc == ZB_OK) {
        for (int r = 0; r < world; ++r) c->ctrl[r] = (ShardCtrl*)peers[r];
        c->peer_ok = true;
    } else if (rc != ZB_ERR_UNSUPPORTED) {
        return fail(rc);
    }
    *out = c;
    return ZB_OK;
}

int zb_shard_comm_destroy(zb_shard_comm* c) {
    if (!c) return ZB_OK;
    cudaDeviceSynchronize();
    for (auto& a : c->allocs) {
        for (int r = 0; r < c->world; ++r)
            if (r != c->rank && a.peer[r]) cudaIpcCloseMemHandle(a.peer[r]);
        if (a.base) cudaFree(a.base);
    }
    for (int r = 0; r < c->world; ++r)
        if (r != c->rank && c->ctrl[r] && c->peer_ok) cudaIpcCloseMemHandle(c->ctrl[r]);
    if (c->ctrl[c->rank]) cudaFree(c->ctrl[c->rank]);
    if (c->staging) cudaFree(c->staging);
    if (c->boot) cudaStreamDestroy(c->boot);
    if (c->nccl) g_nccl.CommDestroy(c->nccl);
    delete c;
    return ZB_OK;
}

int zb_shard_comm_info(const zb_shard_comm* c, int* rank, int* world, int* peer_access) {
    if (!c) return ZB_ERR_INVALID_ARGUMENT;
    if (rank) *rank = c->rank;
    if (world) *world = c->world;
    if (peer_access) *peer_access = c->peer_ok ? 1 : 0;
    return ZB_OK;
}

int zb_shard_status(zb_shard_comm* c, zb_stream s) {
    if (!c) return ZB_ERR_INVALID_ARGUMENT;
    unsigned err = 0;
    ZB_CUDA(cudaStreamSynchronize((cudaStream_t)s));
    ZB_CUDA(cudaMemcpy(&err, &c->ctrl[c->rank]->error, sizeof(err), cudaMemcpyDeviceToHost));
    if (err) {
        snprintf(t_last_error, sizeof(t_last_error), "a row neighbour never signalled (rank %d of %d, op %llu)", c->rank, c->world, c->epoch);
        return ZB_ERR_DEVICE_FAILURE;
    }
    return ZB_OK;
}

int zb_shard_alloc(zb_shard_comm* c, size_t bytes, void** out) {
    if (!c || !out) return ZB_ERR_INVALID_ARGUMENT;
    if (bytes == 0) bytes = 16;
    void* p = nullptr;
    ZB_CUDA(cudaMalloc(&p, bytes));   // plain cudaMalloc: exportable through cudaIpcGetMemHandle (pool memory is not)
    zb_shard_alloc_rec rec;
    rec.base = p;
    rec.bytes = bytes;
    rec.peer[c->rank] = p;
    if (c->world > 1 && c->peer_ok) {
        int rc = exchange_ipc(c, p, rec.peer);
        if (rc != ZB_OK) { cudaFree(p); return rc == ZB_ERR_UNSUPPORTED ? ZB_ERR_DEVICE_FAILURE : rc; }
    }
    c->allocs.push_back(rec);
    *out = p;
    return ZB_OK;
}

int zb_shard_free(zb_shard_comm* c, void* p) {
    if (!c) return ZB_ERR_INVALID_ARGUMENT;
    if (!p) return ZB_OK;
    int idx = -1;
    const zb_shard_alloc_rec* a = find_alloc(c, p, &idx);
    if (!a || a->base != p) return ZB_ERR_INVALID_ARGUMENT;
    ZB_CUDA(cudaDeviceSynchronize());
    if (c->world > 1) {   // nobody may still be reading it: a collective point
        int one = 1, all[ZB_SHARD_MAX_WORLD];
        int rc = gather_host(c, &one, sizeof(int), all);
        if (rc) return rc;
    }
    for (int r = 0; r < c->world; ++r)
        if (r != c->rank && a->peer[r]) cudaIpcCloseMemHandle(a->peer[r]);
    if (c->world > 1) {
        int one = 1, all[ZB_SHARD_MAX_WORLD];
        int rc = gather_host(c, &one, sizeof(int), all);   // every mapping is closed before the owner frees
        if (rc) return rc;
    }
    ZB_CUDA(cudaFree(a->base));
    c->allocs[idx] = zb_shard_alloc_rec();
    return ZB_OK;
}

int zb_shard_image_create(zb_shard_comm* c, const zb_image* block, uint32_t halo_cap, int pixfmt, zb_shard_image** out) {
    if (!c || !block || !out) return ZB_ERR_INVALID_ARGUMENT;
    const size_t pb = pixel_bytes(pixfmt);
    if (pb == 0) return ZB_ERR_UNSUPPORTED;
    int idx = -1;
    const zb_shard_alloc_rec* a = find_alloc(c, block->data, &idx);
    struct Msg { int alloc; int pixfmt; uint32_t rows, cols, halo_cap; uint64_t stride, offset, alloc_bytes; int ok; };
    Msg mine;
    memset(&mine, 0, sizeof(mine));
    mine.ok = a ? 1 : 0;
    if (a) {
        const size_t off = (const char*)block->data - (const char*)a->base;
        const size_t lo = (size_t)halo_cap * block->stride * pb;
        const size_t span_rows = (size_t)block->rows + halo_cap;
        const size_t hi = off + (span_rows ? ((span_rows - 1) * block->stride + block->cols) * pb : 0);
        if (off < lo || hi > a->bytes || block->stride < block->cols) mine.ok = 0;   // the block and its halo rows must lie inside the allocation
        mine.alloc = idx;
        mine.offset = off;
        mine.alloc_bytes = a->bytes;
    }
    mine.pixfmt = pixfmt;
    mine.rows = block->rows;
    mine.cols = block->cols;
    mine.halo_cap = halo_cap;
    mine.stride = block->stride;
    std::vector<Msg> all(c->world);
    int rc = gather_host(c, &mine, sizeof(Msg), all.data());
    if (rc) return rc;
    for (int r = 0; r < c->world; ++r) {
        if (!all[r].ok) return ZB_ERR_INVALID_ARGUMENT;
        if (all[r].pixfmt != pixfmt || all[r].cols != block->cols || all[r].alloc != idx) return ZB_ERR_DIMENSION_MISMATCH;
    }
    zb_shard_image* img = new zb_shard_image();
    memset(img, 0, sizeof(*img));
    img->comm = c;
    img->pixfmt = pixfmt;
    img->cols = block->cols;
    img->halo_cap = halo_cap;
    for (int r = 0; r < c->world; ++r) {
        img->rows[r] = all[r].rows;
        img->stride[r] = all[r].stride;
        void* base = r == c->rank ? a->base : a->peer[r];
        img->data[r] = base ? (char*)base + all[r].offset : nullptr;
    }
    *out = img;
    return ZB_OK;
}

int zb_shard_image_destroy(zb_shard_image* img) {
    delete img;
    return ZB_OK;
}

int zb_shard_image_block(const zb_shard_image* img, zb_image* block) {
    if (!img || !block) return ZB_ERR_INVALID_ARGUMENT;
    const int r = img->comm->rank;
    block->data = img->data[r];
    block->rows = img->rows[r];
    block->cols = img->cols;
    block->stride = img->stride[r];
    return ZB_OK;
}

int zb_shard_split(uint32_t n_items, int rank, int world, uint32_t* lo, uint32_t* hi) {
    if (world < 1 || rank < 0 || rank >= world || !lo || !hi) return ZB_ERR_INVALID_ARGUMENT;
    const uint32_t base = n_items / (uint32_t)world, rem = n_items % (uint32_t)world;
    const uint32_t r = (uint32_t)rank;
    *lo = r * base + (r < rem ? r : rem);
    *hi = *lo + base + (r < rem ? 1u : 0u);
    return ZB_OK;
}

int zb_shard_view(const zb_shard_image* img, uint32_t reach, int border, zb_image* view, uint32_t* interior_first) {
    if (!img || !view) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    return view_of(img, reach, border, view, interior_first);
}

int zb_shard_halo_exchange(zb_shard_comm* c, zb_shard_image* img, uint32_t reach, int border, zb_stream stream) {
    if (!c || !img || img->comm != c) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    if (c->world == 1 || reach == 0) return ZB_OK;
    if (reach > img->halo_cap) return ZB_ERR_INVALID_ARGUMENT;
    cudaStream_t s = (cudaStream_t)stream;
    int up, down;
    neighbours(c, border, &up, &down);
    const size_t pb = pixel_bytes(img->pixfmt);
    const int me = c->rank;
    if ((up >= 0 && img->rows[up] < reach) || (down >= 0 && img->rows[down] < reach) || img->rows[me] < reach) return ZB_ERR_UNSUPPORTED;
    char* mine = (char*)img->data[me];
    const size_t pitch = img->stride[me] * pb;
    const int path = g_shard_path.load();
    if (c->peer_ok && path != 1) {
        PullParams p;
        memset(&p, 0, sizeof(p));
        shard_link(c, border, true, &p.link, nullptr, nullptr);
        p.reach = (int)reach;
        p.row_bytes = (size_t)img->cols * pb;
        p.dst_pitch = pitch;
        p.top_halo = mine - (size_t)reach * pitch;
        p.bottom_halo = mine + (size_t)img->rows[me] * pitch;
        if (up >= 0) {
            p.src_up_pitch = img->stride[up] * pb;
            p.up_rows_src = (const char*)img->data[up] + (size_t)(img->rows[up] - reach) * p.src_up_pitch;
        }
        if (down >= 0) {
            p.src_down_pitch = img->stride[down] * pb;
            p.down_rows_src = (const char*)img->data[down];
        }
        const size_t work = p.row_bytes * reach / 16 + 1;
        const unsigned blocks = (unsigned)std::min<size_t>(64, (work + 255) / 256);
        halo_pull_kernel<<<blocks, 256, 0, s>>>(p);
        ZB_LAUNCHED();
        t_last_kernel = "shard_halo_pull";
        return ZB_OK;
    }
    // fallback: one grouped NCCL send/recv pair per neighbour (no IPC peer mappings on this system)
    if (img->stride[me] != img->cols) return ZB_ERR_UNSUPPORTED;   // whole rows are sent as one contiguous run
    const size_t n = (size_t)reach * pitch;
    ZB_NCCL(g_nccl.GroupStart());
    // order matters when up == down (wrap with 2 ranks): the k-th send to a peer pairs with that peer's k-th recv
    if (up >= 0) ZB_NCCL(g_nccl.Send(mine, n, kNcclUint8, up, c->nccl, s));
    if (down >= 0) ZB_NCCL(g_nccl.Recv(mine + (size_t)img->rows[me] * pitch, n, kNcclUint8, down, c->nccl, s));
    if (down >= 0) ZB_NCCL(g_nccl.Send(mine + (size_t)(img->rows[me] - reach) * pitch, n, kNcclUint8, down, c->nccl, s));
    if (up >= 0) ZB_NCCL(g_nccl.Recv(mine - n, n, kNcclUint8, up, c->nccl, s));
    ZB_NCCL(g_nccl.GroupEnd());
    t_last_kernel = "shard_halo_nccl";
    return ZB_OK;
}

int zb_shard_conv_separable(zb_shard_comm* c, const zb_shard_image* src, zb_shard_image* dst, const float* kx, int nx, const float* ky, int ny,
                            int border, zb_stream stream) {
    if (!c || !src || !dst || src->comm != c || dst->comm != c) return ZB_ERR_INVALID_ARGUMENT;
    if (nx <= 0 || ny <= 0 || !kx || !ky) return ZB_ERR_INVALID_ARGUMENT;
    if (border < ZB_BORDER_ZERO || border > ZB_BORDER_WRAP) return ZB_ERR_INVALID_ARGUMENT;
    const int me = c->rank;
    if (src->pixfmt != dst->pixfmt || src->cols != dst->cols || src->rows[me] != dst->rows[me]) return ZB_ERR_DIMENSION_MISMATCH;
    cudaStream_t s = (cudaStream_t)stream;
    zb_image sblk, dblk;
    zb_shard_image_block(src, &sblk);
    zb_shard_image_block(dst, &dblk);
    if (sblk.rows == 0 || sblk.cols == 0) return ZB_OK;
    const int pixfmt = src->pixfmt;
    if (c->world == 1) return zb_conv_separable(&sblk, &dblk, pixfmt, kx, nx, ky, ny, border, stream);
    const uint32_t half = (uint32_t)(ny / 2);
    int up, down;
    neighbours(c, border, &up, &down);
    const int path = g_shard_path.load();
    if (pixfmt == ZB_PIX_RGBAF32 && c->peer_ok && path == 0 && !g_force_generic.load()) {
        PeerBlock pu{nullptr, 0, 0}, pd{nullptr, 0, 0};
        if (up >= 0) pu = PeerBlock{src->data[up], src->rows[up], src->stride[up]};
        if (down >= 0) pd = PeerBlock{src->data[down], src->rows[down], src->stride[down]};
        // every rank must take the same decision: it depends only on quantities all ranks know (block heights, alignment)
        bool all_fused = true;
        for (int r = 0; r < c->world; ++r)
            all_fused &= src->rows[r] % 8 == 0 && src->rows[r] >= 16 && (((uintptr_t)src->data[r] | (uintptr_t)dst->data[r]) & 15u) == 0;
        all_fused &= src->halo_cap >= 8;   // the kernel's TMA chunks are 8 rows: the halo rows it copies into must exist
        all_fused &= src->cols >= 16 && nx / 2 <= 8 && ny / 2 <= 8 && (nx / 2 >= 1 || ny / 2 >= 1);
        for (int i = 0; i < nx; ++i) all_fused &= !(fabsf(kx[i]) < 1e-10f);
        for (int i = 0; i < ny; ++i) all_fused &= !(fabsf(ky[i]) < 1e-10f);
        if (all_fused) {
            ShardLink link;
            shard_link(c, border, true, &link, nullptr, nullptr);
            int rc = conv_separable_fused_rgbaf32_shard(&sblk, &dblk, kx, nx, ky, ny, border, g_exact_f32.load() != 0, pu, pd, src->halo_cap, link, s);
            if (rc != ZB_ERR_UNSUPPORTED) return rc;
            --c->epoch;   // nothing was launched
            return ZB_ERR_DEVICE_FAILURE;   // the ranks would diverge: report instead of silently taking another path
        }
    }
    // every other configuration: fetch the neighbours' rows into the halo rows, then the ordinary kernels on the extended block
    if (half > src->halo_cap || half > dst->halo_cap) return ZB_ERR_INVALID_ARGUMENT;
    int rc = zb_shard_halo_exchange(c, const_cast<zb_shard_image*>(src), half, border, stream);
    if (rc) return rc;
    zb_image sv, dv;
    uint32_t first = 0;
    if ((rc = view_of(src, half, border, &sv, &first))) return rc;
    // dst rows outside the block are never written (the row window below), so its view may start before its allocation
    dv.data = (char*)dblk.data - (size_t)first * dblk.stride * pixel_bytes(pixfmt);
    dv.rows = sv.rows;
    dv.cols = sv.cols;
    dv.stride = dblk.stride;
    return zb_conv_separable_rows(&sv, &dv, pixfmt, kx, nx, ky, ny, border, first, first + sblk.rows, stream);
}

int zb_shard_gaussian_blur(zb_shard_comm* c, const zb_shard_image* src, zb_shard_image* dst, float sigma, zb_stream stream) {
    if (!c || !src || !dst) return ZB_ERR_INVALID_ARGUMENT;
    if (sigma == 0) {
        zb_image a, b;
        zb_shard_image_block(src, &a);
        zb_shard_image_block(dst, &b);
        return zb_copy(&a, &b, src->pixfmt, stream);
    }
    if (!(sigma > 0) || !std::isfinite(sigma)) return ZB_ERR_INVALID_SIGMA;
    float taps[2048];
    int n = 0;
    int rc = zb_gaussian_taps(sigma, taps, 2048, &n);
    if (rc) return rc;
    return zb_shard_conv_separable(c, src, dst, taps, n, taps, n, ZB_BORDER_MIRROR, stream);
}

int zb_shard_allreduce(zb_shard_comm* c, void* dev_buf, size_t count, int dtype, zb_stream s) {
    return shard_allreduce(c, dev_buf, count, dtype, (cudaStream_t)s);
}

int zb_shard_tune_path(int path) {
    if (path < 0 || path > 2) return ZB_ERR_INVALID_ARGUMENT;
    g_shard_path.store(path);
    return ZB_OK;
}

}  // extern "C"
