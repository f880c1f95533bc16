// comm.cu -- the multi-GPU half of the C ABI (include/phant_gpu.h "multi-GPU"): SURVEY.md 8e behind the boundary, so that
// a Zig host (src/main.zig:143-149 worker threads, one context each) reaches it without Python.
//
// Proofs shard by contiguous, 64-aligned index range; a rank hashes and walks only its shard; the per-batch exchange is
// the accept bitmap (1 bit per proof).  Two transports, same result:
//
//   NCCL    ncclAllGather of every rank's words, issued on the context's own COMM STREAM behind an event, so the next
//           batch's Keccak launch never waits for a peer; the walk that next writes the same destination buffer waits for
//           exactly that collective (callers that alternate two buffers never wait in steady state).
//   peer    (phant_gpu_comm_enable_peer; same node, one process per GPU) the walk kernel's epilogue stores each ballot word
//           straight into every rank's bitmap through NVLink peer mappings (cudaIpc), followed by one flag store per peer
//           from the last CTA; there is no collective launch at all -- a small kernel on the comm stream waits on the flags
//           and copies the gathered bitmap out.
//
// NCCL is dlopen'ed (libnccl.so.2): a single-GPU user of libphantgpu.so has no NCCL dependency, and inside a torch process
// the already loaded copy is reused.  Every failure maps to PHANT_GPU_E_COMM with the NCCL text in phant_gpu_last_error.
#include "../../include/phant_gpu.h"
#include "common.cuh"
#include "ctx.cuh"

#include <dlfcn.h>
#include <unistd.h>
#include <new>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>

using namespace phant;

#define CU(expr)                                                              \
    do {                                                                      \
        cudaError_t e_ = (expr);                                              \
        if (e_ != cudaSuccess) return ctx->fail(e_, #expr, __FILE__, __LINE__); \
    } while (0)

namespace {

struct NcclApi {
    void* handle = nullptr;
    char why[200] = {0};
    ncclResult_t (*GetVersion)(int*) = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi* nccl_api()
{
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {getenv("PHANT_GPU_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n || !*n) continue;
            api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
            snprintf(api.why, sizeof api.why, "dlopen(%s): %s", n, dlerror());
        }
        if (!api.handle) return;
#define SYM(field, name)                                                                  \
    do {                                                                                  \
        *(void**)(&api.field) = dlsym(api.handle, name);                                  \
        if (!api.field) { snprintf(api.why, sizeof api.why, "libnccl lacks %s", name); api.handle = nullptr; return; } \
    } while (0)
        SYM(GetVersion, "ncclGetVersion");
        SYM(GetUniqueId, "ncclGetUniqueId");
        SYM(CommInitRank, "ncclCommInitRank");
        SYM(CommInitAll, "ncclCommInitAll");
        SYM(CommDestroy, "ncclCommDestroy");
        SYM(AllGather, "ncclAllGather");
        SYM(AllReduce, "ncclAllReduce");
        SYM(Broadcast, "ncclBroadcast");
        SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
    });
    return api.handle ? &api : nullptr;
}

int comm_fail(phant_gpu_ctx* ctx, ncclResult_t r, const char* what)
{
    NcclApi* api = nccl_api();
    snprintf(ctx->last_error, sizeof ctx->last_error, "NCCL: %s: %s", what, api ? api->GetErrorString(r) : "library not loaded");
    return PHANT_GPU_E_COMM;
}
#define NC(expr)                                                       \
    do {                                                               \
        ncclResult_t r_ = (expr);                                      \
        if (r_ != ncclSuccess) return comm_fail(ctx, r_, #expr);       \
    } while (0)

int comm_streams(phant_gpu_ctx* ctx)
{
    if (!ctx->comm_stream) CU(cudaStreamCreateWithFlags(&ctx->comm_stream, cudaStreamNonBlocking));
    if (!ctx->ev_compute) CU(cudaEventCreateWithFlags(&ctx->ev_compute, cudaEventDisableTiming));
    if (!ctx->h_comm) CU(cudaMallocHost(&ctx->h_comm, 16384));
    return PHANT_GPU_OK;
}

// the event that marks "the last collective touching `buf` is done" (one per distinct destination buffer, at most 8 kept)
cudaEvent_t fence_for(phant_gpu_ctx* ctx, const void* buf)
{
    for (auto& f : ctx->fence_events)
        if (f.buf == buf) return f.ev;
    if (ctx->fence_events.size() >= 8) { // recycle the oldest entry: wait for it once, then reuse its event
        phant_gpu_ctx::Fence f = ctx->fence_events.front();
        ctx->fence_events.erase(ctx->fence_events.begin());
        cudaStreamWaitEvent(ctx->stream, f.ev, 0);
        f.buf = buf;
        ctx->fence_events.push_back(f);
        return f.ev;
    }
    cudaEvent_t ev = nullptr;
    if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    ctx->fence_events.push_back({buf, ev});
    return ev;
}

__global__ void reject_count_kernel(const uint8_t* __restrict__ status, const uint32_t* __restrict__ block_of_proof, uint64_t n, uint64_t n_blocks,
                                    uint32_t* __restrict__ counts)
{
    for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t st = status[p];
        const uint32_t b = block_of_proof[p];
        if (st != 1 && st != 2 && b < n_blocks) atomicAdd(&counts[b], 1u); // reject (0) or missing node (3)
    }
}

} // namespace

// ------------------------------------------------------------------------------------------------
// peer transport: one symmetric region per rank, mapped into every rank of the node
// ------------------------------------------------------------------------------------------------
// region layout: [ready[2][16] u64][done[2][16] u64][err u32, tickets ...] (1 KB header) then 2 gathered-bitmap buffers.
// ready[b][src] = last step whose words rank `src` has stored into MY buffer b; done[b][src] = last step of buffer b that
// rank `src` has copied out of ITS buffer b (so I may overwrite it).  Steps count from 1; step s uses buffer s & 1.
struct phant_gpu_ctx::Peer {
    int world = 0, rank = 0;
    uint64_t cap_words = 0;            // per buffer
    uint8_t* region[PEER_MAX_WORLD] = {}; // every rank's region as mapped here (region[rank] = my own allocation)
    bool ipc_opened[PEER_MAX_WORLD] = {};
    uint64_t step = 0;
    bool usable = false;               // set once every rank has mapped every region (a half-built object is only ever released)
    static constexpr size_t HDR = 1024;
    unsigned long long* ready(int r, int b, int src) const { return (unsigned long long*)region[r] + (b * PEER_MAX_WORLD + src); }
    unsigned long long* done(int r, int b, int src) const { return (unsigned long long*)region[r] + (2 * PEER_MAX_WORLD + b * PEER_MAX_WORLD + src); }
    uint32_t* err(int r) const { return (uint32_t*)(region[r] + 8 * 4 * PEER_MAX_WORLD); }
    uint32_t* ticket(int which) const { return err(rank) + 4 + which; } // my own region only
    uint64_t* bitmap(int r, int b) const { return (uint64_t*)(region[r] + HDR) + (uint64_t)b * cap_words; }
};

namespace {
struct PeerRec { cudaIpcMemHandle_t h; uint64_t pid; uint64_t ptr; int32_t dev; int32_t pad; };

void peer_release(phant_gpu_ctx* ctx)
{
    phant_gpu_ctx::Peer* p = ctx->peer;
    if (!p) return;
    for (int r = 0; r < p->world; ++r)
        if (r != p->rank && p->ipc_opened[r]) cudaIpcCloseMemHandle(p->region[r]);
    if (p->region[p->rank]) cudaFree(p->region[p->rank]);
    delete p;
    ctx->peer = nullptr;
}
} // namespace

// the walk that is about to write `walk_fence_buf` waits (on the device) for the collective still using that buffer
int phant_gpu_ctx::wait_walk_fence()
{
    phant_gpu_ctx* ctx = this;
    if (!walk_fence_buf) return PHANT_GPU_OK;
    for (auto& f : fence_events)
        if (f.buf == walk_fence_buf) CU(cudaStreamWaitEvent(stream, f.ev, 0));
    walk_fence_buf = nullptr;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_shard_range(uint64_t n, int rank, int world, uint64_t* lo, uint64_t* hi)
{
    if (!lo || !hi || world < 1 || rank < 0 || rank >= world) return PHANT_GPU_E_INVALID;
    const uint64_t per = ((n + world - 1) / world + 63) / 64 * 64;
    *lo = (uint64_t)rank * per < n ? (uint64_t)rank * per : n;
    *hi = *lo + per < n ? *lo + per : n;
    return PHANT_GPU_OK;
}

extern "C" uint64_t phant_gpu_sharded_bitmap_words(uint64_t n, int world)
{
    if (world < 1) return 0;
    const uint64_t per = ((n + world - 1) / world + 63) / 64 * 64;
    return (per / 64) * (uint64_t)world;
}

extern "C" int phant_gpu_comm_get_unique_id(uint8_t id[PHANT_GPU_COMM_ID_BYTES])
{
    if (!id) return PHANT_GPU_E_INVALID;
    NcclApi* api = nccl_api();
    if (!api) return PHANT_GPU_E_COMM;
    ncclUniqueId u;
    static_assert(sizeof u == PHANT_GPU_COMM_ID_BYTES, "unique id size");
    if (api->GetUniqueId(&u) != ncclSuccess) return PHANT_GPU_E_COMM;
    memcpy(id, &u, sizeof u);
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_comm_init(phant_gpu_ctx* ctx, const uint8_t id[PHANT_GPU_COMM_ID_BYTES], int rank, int world)
{
    if (!ctx || !id || world < 1 || rank < 0 || rank >= world || ctx->comm) return PHANT_GPU_E_INVALID;
    NcclApi* api = nccl_api();
    if (!api) {
        snprintf(ctx->last_error, sizeof ctx->last_error, "NCCL not loadable: %s", nccl_api() ? "" : "libnccl.so.2 (set PHANT_GPU_NCCL_LIB)");
        return PHANT_GPU_E_COMM;
    }
    CU(cudaSetDevice(ctx->device));
    if (int rc = comm_streams(ctx)) return rc;
    ncclUniqueId u;
    memcpy(&u, id, sizeof u);
    ncclComm_t c = nullptr;
    NC(api->CommInitRank(&c, world, u, rank));
    ctx->comm = c;
    ctx->comm_rank = rank;
    ctx->comm_world = world;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_comm_init_local(phant_gpu_ctx** ctxs, int n)
{
    if (!ctxs || n < 1 || n > 64) return PHANT_GPU_E_INVALID;
    for (int i = 0; i < n; ++i)
        if (!ctxs[i] || ctxs[i]->comm) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = ctxs[0];
    NcclApi* api = nccl_api();
    if (!api) { snprintf(ctx->last_error, sizeof ctx->last_error, "NCCL not loadable (libnccl.so.2; PHANT_GPU_NCCL_LIB overrides)"); return PHANT_GPU_E_COMM; }
    int devs[64];
    ncclComm_t comms[64];
    for (int i = 0; i < n; ++i) devs[i] = ctxs[i]->device;
    NC(api->CommInitAll(comms, n, devs));
    for (int i = 0; i < n; ++i) {
        ctxs[i]->comm = comms[i];
        ctxs[i]->comm_rank = i;
        ctxs[i]->comm_world = n;
        if (cudaSetDevice(ctxs[i]->device) != cudaSuccess) return PHANT_GPU_E_CUDA;
        if (int rc = comm_streams(ctxs[i])) return rc;
    }
    return PHANT_GPU_OK;
}

// collective: back to the NCCL gather (barrier first: nobody unmaps a region a peer's kernels could still be storing into)
extern "C" int phant_gpu_comm_disable_peer(phant_gpu_ctx* ctx)
{
    if (!ctx) return PHANT_GPU_E_INVALID;
    if (!ctx->peer) return PHANT_GPU_OK;
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->comm_stream) CU(cudaStreamSynchronize(ctx->comm_stream));
    NcclApi* api = nccl_api();
    if (api && ctx->comm && ctx->d_comm.ptr) {
        NC(api->AllReduce(ctx->d_comm.ptr, ctx->d_comm.ptr, 1, ncclInt32, ncclMin, (ncclComm_t)ctx->comm, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    peer_release(ctx);
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_comm_peer_status(phant_gpu_ctx* ctx, int* enabled, uint64_t* steps, int* timed_out)
{
    if (!ctx) return PHANT_GPU_E_INVALID;
    if (enabled) *enabled = ctx->peer && ctx->peer->usable ? 1 : 0;
    if (steps) *steps = ctx->peer && ctx->peer->usable ? ctx->peer->step : 0;
    if (timed_out) {
        *timed_out = 0;
        if (ctx->peer && ctx->peer->usable) {
            CU(cudaSetDevice(ctx->device));
            uint32_t e = 0;
            CU(cudaMemcpy(&e, ctx->peer->err(ctx->peer->rank), 4, cudaMemcpyDeviceToHost));
            *timed_out = (int)e;
        }
    }
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_comm_info(const phant_gpu_ctx* ctx, int* rank, int* world, int* nccl_version)
{
    if (!ctx) return PHANT_GPU_E_INVALID;
    if (rank) *rank = ctx->comm_rank;
    if (world) *world = ctx->comm_world;
    if (nccl_version) {
        *nccl_version = 0;
        NcclApi* api = nccl_api();
        if (api) api->GetVersion(nccl_version);
    }
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_comm_destroy(phant_gpu_ctx* ctx)
{
    if (!ctx) return PHANT_GPU_E_INVALID;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->comm_stream) cudaStreamSynchronize(ctx->comm_stream);
    if (ctx->peer) {
        // nobody may unmap or free a region a peer's kernels could still be storing into: one collective as the barrier
        NcclApi* api = nccl_api();
        if (api && ctx->comm && ctx->d_comm.ptr) {
            api->AllReduce(ctx->d_comm.ptr, ctx->d_comm.ptr, 1, ncclInt32, ncclMin, (ncclComm_t)ctx->comm, ctx->stream);
            cudaStreamSynchronize(ctx->stream);
        }
        peer_release(ctx);
    }
    if (ctx->comm) {
        NcclApi* api = nccl_api();
        if (api) api->CommDestroy((ncclComm_t)ctx->comm);
        ctx->comm = nullptr;
    }
    for (auto& f : ctx->fence_events) cudaEventDestroy(f.ev);
    ctx->fence_events.clear();
    if (ctx->ev_compute) { cudaEventDestroy(ctx->ev_compute); ctx->ev_compute = nullptr; }
    if (ctx->comm_stream) { cudaStreamDestroy(ctx->comm_stream); ctx->comm_stream = nullptr; }
    if (ctx->h_comm) { cudaFreeHost(ctx->h_comm); ctx->h_comm = nullptr; }
    ctx->comm_rank = 0;
    ctx->comm_world = 1;
    return PHANT_GPU_OK;
}

// make the context's stream wait (on the device) for every collective issued so far; then anything the caller enqueues on
// that stream -- or phant_gpu_synchronize -- sees the gathered results
extern "C" int phant_gpu_comm_fence(phant_gpu_ctx* ctx)
{
    if (!ctx) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    for (auto& f : ctx->fence_events) CU(cudaStreamWaitEvent(ctx->stream, f.ev, 0));
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_comm_enable_peer(phant_gpu_ctx* ctx, uint64_t max_n_global)
{
    if (!ctx || max_n_global == 0) return PHANT_GPU_E_INVALID;
    if (ctx->peer && ctx->peer->usable) return PHANT_GPU_OK;
    if (ctx->peer) peer_release(ctx); // left over from a failed attempt
    const int world = ctx->comm_world, rank = ctx->comm_rank;
    NcclApi* api = nccl_api();
    if (world < 2 || world > PEER_MAX_WORLD || !api || !ctx->comm) { snprintf(ctx->last_error, sizeof ctx->last_error, "peer transport needs a communicator of 2..16 ranks"); return PHANT_GPU_E_COMM; }
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    auto* p = new (std::nothrow) phant_gpu_ctx::Peer();
    if (!p) return PHANT_GPU_E_OOM;
    p->world = world; p->rank = rank;
    p->cap_words = phant_gpu_sharded_bitmap_words(max_n_global, world);
    const size_t bytes = phant_gpu_ctx::Peer::HDR + 2 * 8 * p->cap_words + 64;
    uint8_t* mine = nullptr;
    int ok_local = 1;
    if (cudaMalloc((void**)&mine, bytes) != cudaSuccess) { cudaGetLastError(); ok_local = 0; mine = nullptr; }
    p->region[rank] = mine;
    ctx->peer = p; // owned by the context from here on: every error return below leaves a non-usable object that
                   // phant_gpu_comm_disable_peer / phant_gpu_comm_destroy release
    PeerRec* h = (PeerRec*)ctx->h_comm;
    static_assert(sizeof(PeerRec) == 88, "record layout");
    if ((size_t)(world + 1) * sizeof(PeerRec) > 16384) { peer_release(ctx); return PHANT_GPU_E_INVALID; }
    memset(h, 0, sizeof(PeerRec));
    if (ok_local) {
        CU(cudaMemsetAsync(mine, 0, bytes, s));
        if (cudaIpcGetMemHandle(&h->h, mine) != cudaSuccess) { cudaGetLastError(); ok_local = 0; }
        h->pid = (uint64_t)getpid(); h->ptr = (uint64_t)(uintptr_t)mine; h->dev = ctx->device;
    }
    h->pad = ok_local;
    if (int rc = ctx->d_comm.reserve(ctx, sizeof(PeerRec) * (world + 1))) { peer_release(ctx); return rc; }
    uint8_t* d = (uint8_t*)ctx->d_comm.ptr;
    CU(cudaMemcpyAsync(d + sizeof(PeerRec) * rank, h, sizeof(PeerRec), cudaMemcpyHostToDevice, s));
    NC(api->AllGather(d + sizeof(PeerRec) * rank, d, sizeof(PeerRec), ncclUint8, (ncclComm_t)ctx->comm, s));
    PeerRec* all = h + 1;
    CU(cudaMemcpyAsync(all, d, sizeof(PeerRec) * world, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    // every rank takes the same decision from the same records; mapping failures are exchanged in a second round
    int ok = 1;
    for (int r = 0; r < world; ++r) ok &= all[r].pad;
    for (int r = 0; ok && r < world; ++r) {
        if (r == rank) continue;
        if (all[r].pid == (uint64_t)getpid()) { // several contexts of ONE process: not supported by this transport (NCCL stays)
            ok = 0;
            break;
        } else {
            void* q = nullptr;
            if (cudaIpcOpenMemHandle(&q, all[r].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
            p->region[r] = (uint8_t*)q;
            p->ipc_opened[r] = true;
        }
    }
    // agree: one all-reduce (min) of the local verdicts, which is also the barrier "every region is zeroed and mapped"
    int32_t* flag = (int32_t*)h;
    *flag = ok;
    CU(cudaMemcpyAsync(d, flag, 4, cudaMemcpyHostToDevice, s));
    NC(api->AllReduce(d, d, 1, ncclInt32, ncclMin, (ncclComm_t)ctx->comm, s));
    CU(cudaMemcpyAsync(flag, d, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (!*flag) {
        peer_release(ctx);
        snprintf(ctx->last_error, sizeof ctx->last_error, "peer mapping (cudaIpc / peer access) not available on every rank");
        return PHANT_GPU_E_COMM;
    }
    p->usable = true;
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// V, sharded
// ------------------------------------------------------------------------------------------------
extern "C" int phant_gpu_verify_proofs_sharded(phant_gpu_ctx* ctx, const phant_gpu_proof_batch* local, uint64_t n_global,
                                               uint64_t* global_bitmap, uint8_t* status, uint64_t* val_off, uint32_t* val_len)
{
    if (!ctx || !local || !global_bitmap) return PHANT_GPU_E_INVALID;
    const int world = ctx->comm_world, rank = ctx->comm_rank;
    uint64_t lo = 0, hi = 0;
    phant_gpu_shard_range(n_global, rank, world, &lo, &hi);
    if (local->n_proofs != hi - lo) return PHANT_GPU_E_INVALID; // the caller shards with phant_gpu_shard_range
    const uint64_t per_words = phant_gpu_sharded_bitmap_words(n_global, world) / world;
    CU(cudaSetDevice(ctx->device));
    NcclApi* api = world > 1 ? nccl_api() : nullptr;
    if (world > 1 && (!api || !ctx->comm)) { snprintf(ctx->last_error, sizeof ctx->last_error, "no communicator"); return PHANT_GPU_E_COMM; }

    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) {
        // asynchronous: Keccak + walk on the context's stream, the gather on the comm stream behind an event
        uint64_t* mine = global_bitmap + (uint64_t)rank * per_words;
        const uint64_t my_words = (hi - lo + 63) / 64;
        phant_gpu_ctx::Peer* pr = ctx->peer;
        // (the choice must be the same on every rank: it depends on n_global and world only -- equal, 64-aligned shards)
        if (world > 1 && pr && pr->usable && n_global && n_global % (64ull * world) == 0 && per_words * world <= pr->cap_words) {
            // ---- peer transport: the walk's epilogue stores into every rank's buffer and publishes the step; the comm stream
            // only waits for the other ranks' words, copies the gathered bitmap out and releases the buffer ----
            NvtxRange nvtx("phant:gather(peer)");
            const unsigned long long step = ++pr->step;
            const int b = (int)(step & 1);
            PeerOut po{};
            for (int r = 0; r < world; ++r) {
                po.dst[r] = (uint32_t*)(pr->bitmap(r, b) + (uint64_t)rank * per_words);
                po.ready[r] = pr->ready(r, b, rank);
            }
            po.done = pr->done(rank, b, 0);
            po.wait_done = step > 2 ? step - 2 : 0;
            po.step = step;
            po.ticket = pr->ticket(0);
            po.err = pr->err(rank);
            po.world = (uint32_t)world;
            ctx->walk_peer = &po;
            const int rc = phant_gpu_verify_proofs(ctx, local, nullptr, status, val_off, val_len);
            ctx->walk_peer = nullptr;
            if (rc) return rc;
            cudaEvent_t done_ev = fence_for(ctx, global_bitmap);
            if (!done_ev) return PHANT_GPU_E_CUDA;
            CU(cudaEventRecord(ctx->ev_compute, ctx->stream));
            CU(cudaStreamWaitEvent(ctx->comm_stream, ctx->ev_compute, 0));
            PeerOut sig{};
            for (int r = 0; r < world; ++r) sig.ready[r] = pr->done(r, b, rank);
            sig.ticket = pr->ticket(1);
            sig.err = pr->err(rank);
            CU(launch_peer_collect(ctx->comm_stream, pr->ready(rank, b, 0), (uint32_t)world, step, pr->bitmap(rank, b), global_bitmap,
                                   8 * per_words * world, sig));
            CU(cudaEventRecord(done_ev, ctx->comm_stream));
            ctx->stats.launches++;
            return PHANT_GPU_OK;
        }
        if (world > 1) ctx->walk_fence_buf = global_bitmap; // the walk waits for the collective that still uses this buffer
        if (local->n_proofs) {
            if (int rc = phant_gpu_verify_proofs(ctx, local, mine, status, val_off, val_len)) return rc;
        } else if (int rc = ctx->wait_walk_fence()) return rc;
        if (world == 1) return PHANT_GPU_OK;
        if (my_words < per_words) CU(cudaMemsetAsync(mine + my_words, 0, 8 * (per_words - my_words), ctx->stream)); // short / empty last shard
        NvtxRange nvtx("phant:gather");
        cudaEvent_t done = fence_for(ctx, global_bitmap);
        if (!done) return PHANT_GPU_E_CUDA;
        CU(cudaEventRecord(ctx->ev_compute, ctx->stream));
        CU(cudaStreamWaitEvent(ctx->comm_stream, ctx->ev_compute, 0));
        NC(api->AllGather(mine, global_bitmap, per_words, ncclUint64, (ncclComm_t)ctx->comm, ctx->comm_stream));
        CU(cudaEventRecord(done, ctx->comm_stream));
        ctx->stats.launches++;
        return PHANT_GPU_OK;
    }

    // host pointers: the library's own device bitmap holds this shard's words after the call below
    if (local->n_proofs)
        if (int rc = phant_gpu_verify_proofs(ctx, local, nullptr, status, val_off, val_len)) return rc;
    const uint64_t my_words = (hi - lo + 63) / 64;
    if (world == 1) {
        if (int rc = copy_out(ctx, global_bitmap, ctx->d_bitmap.ptr, 8 * my_words)) return rc;
        CU(cudaStreamSynchronize(ctx->stream));
        return PHANT_GPU_OK;
    }
    if (int rc = ctx->d_comm.reserve(ctx, 8 * per_words * world)) return rc;
    uint64_t* g = (uint64_t*)ctx->d_comm.ptr;
    CU(cudaMemsetAsync(g + (uint64_t)rank * per_words, 0, 8 * per_words, ctx->stream));
    if (my_words) CU(cudaMemcpyAsync(g + (uint64_t)rank * per_words, ctx->d_bitmap.ptr, 8 * my_words, cudaMemcpyDeviceToDevice, ctx->stream));
    NC(api->AllGather(g + (uint64_t)rank * per_words, g, per_words, ncclUint64, (ncclComm_t)ctx->comm, ctx->stream));
    if (int rc = copy_out(ctx, global_bitmap, g, 8 * per_words * world)) return rc;
    ctx->stats.launches++;
    CU(cudaStreamSynchronize(ctx->stream));
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// per-block reject counts (config C5: blocks sharded, per-block accept = no rejected proof), one all-reduce
// ------------------------------------------------------------------------------------------------
extern "C" int phant_gpu_block_reject_counts(phant_gpu_ctx* ctx, const uint8_t* status, const uint32_t* block_of_proof, uint64_t n_proofs,
                                             uint64_t n_blocks, uint32_t* counts)
{
    if (!ctx || !counts || (n_proofs && (!status || !block_of_proof)) || n_blocks == 0) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool dev = ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS;
    const uint8_t* d_status = status; const uint32_t* d_map = block_of_proof; uint32_t* d_counts = counts;
    if (!dev) {
        uint32_t* m;
        uint8_t* st;
        if (int rc = carve(ctx, ctx->d_rej, [&](Carve& c) { d_counts = c.take<uint32_t>(n_blocks); m = c.take<uint32_t>(n_proofs); st = c.take<uint8_t>(n_proofs); }))
            return rc;
        if (n_proofs) {
            CU(cudaMemcpyAsync(m, block_of_proof, 4 * n_proofs, cudaMemcpyHostToDevice, s));
            CU(cudaMemcpyAsync(st, status, n_proofs, cudaMemcpyHostToDevice, s));
            ctx->stats.h2d_bytes += 5 * n_proofs;
        }
        d_map = m; d_status = st;
    }
    CU(cudaMemsetAsync(d_counts, 0, 4 * n_blocks, s));
    if (n_proofs) {
        uint64_t blocks = (n_proofs + 255) / 256;
        const uint64_t cap = (uint64_t)keccak_num_sms(ctx->device) * 8;
        if (blocks > cap) blocks = cap;
        reject_count_kernel<<<(unsigned)blocks, 256, 0, s>>>(d_status, d_map, n_proofs, n_blocks, d_counts);
        CU(cudaGetLastError());
        ctx->stats.launches++;
    }
    if (ctx->comm_world > 1) {
        NcclApi* api = nccl_api();
        if (!api || !ctx->comm) { snprintf(ctx->last_error, sizeof ctx->last_error, "no communicator"); return PHANT_GPU_E_COMM; }
        NC(api->AllReduce(d_counts, d_counts, n_blocks, ncclUint32, ncclSum, (ncclComm_t)ctx->comm, s));
        ctx->stats.launches++;
    }
    if (dev) return PHANT_GPU_OK;
    if (int rc = copy_out(ctx, counts, d_counts, 4 * n_blocks)) return rc;
    CU(cudaStreamSynchronize(s));
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// S, sharded by the top nibble of keccak(address): subtree roots here, one all-gather, root branch hashed on every rank
// ------------------------------------------------------------------------------------------------
extern "C" int phant_gpu_nibble_owner(int nibble, int world) { return world < 1 ? 0 : nibble * (world < 16 ? world : 16) / 16; }

extern "C" int phant_gpu_state_root_sharded(phant_gpu_ctx* ctx, const phant_gpu_accounts* mine, uint8_t out_root[32])
{
    if (!ctx || !mine || !out_root) return PHANT_GPU_E_INVALID;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // host tables only (as phant_gpu_state_root)
    const int world = ctx->comm_world, rank = ctx->comm_rank;
    if (world == 1) return phant_gpu_state_root(ctx, mine, out_root);
    NcclApi* api = nccl_api();
    if (!api || !ctx->comm) { snprintf(ctx->last_error, sizeof ctx->last_error, "no communicator"); return PHANT_GPU_E_COMM; }
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    // record = 16 x 32 subtree hashes + mask (4) + account count (8) + padding -> 528 bytes per rank
    constexpr size_t REC = 528;
    struct Rec { uint8_t roots[512]; uint32_t mask; uint32_t pad; uint64_t n_accounts; };
    static_assert(sizeof(Rec) == REC, "record layout");
    if ((size_t)(world + 1) * REC > 16384) return PHANT_GPU_E_INVALID; // pinned staging area: my record + every rank's
    Rec* h = (Rec*)ctx->h_comm;
    memset(h, 0, REC);
    if (mine->n_accounts) {
        if (int rc = phant_gpu_state_subtree_roots(ctx, mine, h->roots, &h->mask)) return rc;
    }
    h->n_accounts = mine->n_accounts;
    if (int rc = ctx->d_comm.reserve(ctx, REC * (world + 1))) return rc;
    uint8_t* d = (uint8_t*)ctx->d_comm.ptr;
    CU(cudaMemcpyAsync(d + REC * rank, h, REC, cudaMemcpyHostToDevice, s));
    NC(api->AllGather(d + REC * rank, d, REC, ncclUint8, (ncclComm_t)ctx->comm, s));
    ctx->stats.launches++;
    Rec* all = (Rec*)((uint8_t*)ctx->h_comm + REC);
    CU(cudaMemcpyAsync(all, d, REC * world, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    uint32_t mask_all = 0;
    int holder = -1, holders = 0;
    for (int r = 0; r < world; ++r) {
        if (all[r].mask & mask_all) { snprintf(ctx->last_error, sizeof ctx->last_error, "two ranks hold accounts of one root-branch slot"); return PHANT_GPU_E_INVALID; }
        mask_all |= all[r].mask;
        if (all[r].n_accounts) { holder = r; ++holders; }
    }
    if (__builtin_popcount(mask_all) < 2) {
        // the root is not a branch (0 or 1 populated slot): the one rank that holds accounts computes the plain root
        if (holders > 1) { snprintf(ctx->last_error, sizeof ctx->last_error, "accounts of one slot spread over ranks"); return PHANT_GPU_E_INVALID; }
        const int root_rank = holder < 0 ? 0 : holder;
        if (rank == root_rank) {
            if (int rc = phant_gpu_state_root(ctx, mine, out_root)) return rc;
            memcpy(h, out_root, 32);
            CU(cudaMemcpyAsync(d, h, 32, cudaMemcpyHostToDevice, s));
        }
        NC(api->Broadcast(d, d, 32, ncclUint8, root_rank, (ncclComm_t)ctx->comm, s));
        CU(cudaMemcpyAsync(h, d, 32, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        memcpy(out_root, h, 32);
        return PHANT_GPU_OK;
    }
    // rlp([ref_0 .. ref_15, ""]) (src/mpt/mpt.zig:218-247): populated slots carry the 32-byte subtree hash (an account leaf
    // is >= 70 bytes, so never embedded), the others and the value the empty string
    uint8_t node[3 + 16 * 33 + 1];
    size_t body = 1;
    for (int v = 0; v < 16; ++v) body += (mask_all >> v) & 1 ? 33 : 1;
    uint8_t* q = node;
    if (body < 56) *q++ = (uint8_t)(0xc0 + body);
    else if (body < 256) { *q++ = 0xf8; *q++ = (uint8_t)body; }
    else { *q++ = 0xf9; *q++ = (uint8_t)(body >> 8); *q++ = (uint8_t)body; }
    for (int v = 0; v < 16; ++v) {
        if ((mask_all >> v) & 1) {
            int owner = -1;
            for (int r = 0; r < world; ++r) if ((all[r].mask >> v) & 1) owner = r;
            *q++ = 0xa0;
            memcpy(q, all[owner].roots + 32 * v, 32);
            q += 32;
        } else *q++ = 0x80;
    }
    *q++ = 0x80;
    const uint64_t off[2] = {0, (uint64_t)(q - node)};
    return phant_gpu_keccak256_batch(ctx, node, off, 1, out_root);
}
