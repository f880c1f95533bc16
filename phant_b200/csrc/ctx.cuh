// ctx.cuh -- the context object behind `phant_gpu_ctx*` (include/phant_gpu.h).
#pragma once
#include "../../include/phant_gpu.h"
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <array>
#include <vector>

#include <nvtx3/nvToolsExt.h>
// NVTX ranges around the phases of a call (H2D staging, hash, walk, gather): free when no tool is attached (header-only
// NVTX v3 resolves its injection library lazily), visible in nsys / ncu --nvtx timelines
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

struct phant_gpu_ctx;

struct DevBuf {
    void* ptr = nullptr;
    size_t cap = 0;
    int reserve(phant_gpu_ctx* ctx, size_t bytes); // grows (never shrinks); contents are not preserved
    void release();
};

// a witness node set hashed once, with its digest -> node table (walk_kernel.cu "bag"): `capacity` slots, a power of two
// >= 2 x the node count and at least 64.  The arrays live in the context's d_digests, d_summary and d_index.
struct NodeTable {
    const uint8_t* digests;
    const uint32_t* summary; // null unless asked for
    const uint32_t* table;
    uint32_t capacity;
};

struct EventPair {
    cudaEvent_t a = nullptr, b = nullptr;
    int which = 0; // 0 keccak, 1 walk
};

struct phant_gpu_ctx {
    int device = 0;
    uint32_t flags = 0;
    cudaStream_t stream = nullptr;     // the stream work is issued on (own_stream unless the caller set one)
    cudaStream_t own_stream = nullptr;
    char last_error[256] = {0};
    phant_gpu_stats stats = {};

    // staging + scratch (device)
    DevBuf d_msgs, d_off, d_out;                                          // K
    // V; both host-pointer paths of V leave the verdict bitmap in d_bitmap, where the sharded host path (comm.cu) reads it
    DevBuf d_first, d_keys, d_roots, d_digests, d_bitmap, d_status, d_voff, d_vlen, d_summary, d_index;
    DevBuf d_idx, d_order, d_cub, d_perms;                                // regrouping
    DevBuf d_synth;                                                       // synth: per-proof counts and their scans
    // the forest builder (trie.cu): scratch sized by the key count, scratch sized by the largest level, the leaves' RLP and
    // one unit pass's RLP
    DevBuf fo_keys, fo_level, fo_leaf_rlp, fo_unit_rlp;
    DevBuf sp_words;                                                      // the sparse trie update's counter words (trie.cu)
    DevBuf st_in, st_hash, st_seg, st_tmp, st_sort, st_acc;               // state-root staging
    DevBuf sr_stage, sr_work;                                             // pre-state reads: host staging; code table and account records
    DevBuf tr_in, tr_keys, tr_sort, tr_front[2], tr_items, tr_work, tr_vals;  // transition roots (trie.cu "T")
    bool perms_init = false, perms_pending = false;

    std::array<DevBuf*, 41> all_bufs()
    {
        return {&d_msgs, &d_off, &d_out, &d_first, &d_keys, &d_roots, &d_digests, &d_bitmap, &d_status, &d_voff, &d_vlen,
                &d_idx, &d_order, &d_cub, &d_perms, &d_synth, &fo_keys, &fo_level, &fo_leaf_rlp, &fo_unit_rlp, &sp_words,
                &st_in, &st_hash, &st_seg, &st_tmp, &st_sort, &st_acc, &d_summary, &d_index, &d_comm, &d_rej,
                &sr_stage, &sr_work, &tr_in, &tr_keys, &tr_sort, &tr_front[0], &tr_front[1], &tr_items, &tr_work, &tr_vals};
    }

    // device timing of the dominant kernels: event pairs recorded on `stream`, resolved lazily
    std::vector<EventPair> pairs; // pool, grows on demand; the first n_pairs are pending
    int n_pairs = 0;
    // host-pointer pipeline: H2D on copy_stream chunk by chunk, kernels on `stream` behind an event per chunk
    cudaStream_t copy_stream = nullptr;
    std::vector<cudaEvent_t> chunk_events;
    // multi-GPU (comm.cu): one NCCL communicator per context, collectives on their own stream so that the next batch's
    // Keccak launch never waits for a peer; `fence_events` remembers, per destination buffer, the collective that still
    // reads / writes it (the walk that next writes that buffer waits for exactly that one)
    void* comm = nullptr;          // ncclComm_t
    int comm_rank = 0, comm_world = 1;
    cudaStream_t comm_stream = nullptr;
    cudaEvent_t ev_compute = nullptr;
    struct Fence { const void* buf; cudaEvent_t ev; };
    std::vector<Fence> fence_events;
    const void* walk_fence_buf = nullptr; // set by the sharded entry point: buffer the next walk launch is about to write
    DevBuf d_comm, d_rej;
    void* h_comm = nullptr;        // small pinned staging area (subtree roots, counters)
    // peer-memory path (comm.cu): symmetric buffers mapped from every rank of the node
    struct Peer;
    Peer* peer = nullptr;
    const void* walk_peer = nullptr; // (const phant::PeerOut*) set by the sharded entry point around one verify call
    int wait_walk_fence();

    void time_begin(int which);
    void time_end();
    void resolve_times();

    int fail(cudaError_t e, const char* what, const char* file, int line);
    int hash_csr(const uint8_t* d_msgs, const uint64_t* d_off, uint64_t n, uint64_t total_bytes, uint8_t* d_out,
                 uint32_t* d_summary = nullptr);
    // a host CSR of n nodes or messages into d_msgs / d_off, d_msgs reserved with extra_bytes behind the bytes; off may be
    // null when n == 0
    int upload_csr(const uint8_t* data, const uint64_t* off, uint64_t n, uint64_t total_bytes, uint64_t extra_bytes);
    // the node set on the device (n <= 2^30) hashed, with summaries when asked, and its digest -> node table built
    int node_table(const uint8_t* d_nodes, const uint64_t* d_off, uint64_t n, uint64_t total_bytes, bool summaries, NodeTable* out);
    // messages in slots: message m = d_msgs[d_off[m] .. d_off[m] + d_len[m]); no regrouping, no statistics pass
    int hash_slots(const uint8_t* d_msgs, const uint64_t* d_off, const uint64_t* d_len, uint64_t n, uint8_t* d_out);
    // chain-form proofs (no node_index) in one fused hash-and-walk kernel, then the verdict pass (abi.cu); fused_ok() says
    // whether this call may take that path
    bool fused_ok(const uint8_t* d_nodes, uint64_t n_proofs, uint64_t n_nodes) const;
    int verify_fused(const uint8_t* d_nodes, const uint64_t* d_node_off, uint64_t n_nodes, uint64_t total_bytes, const uint64_t* d_proof_first,
                     uint64_t n_proofs, const uint8_t* d_keys, const uint8_t* d_roots, uint64_t n_roots, uint64_t* d_bitmap /*nullable*/,
                     uint8_t* d_status /*nullable*/, uint64_t* d_voff /*nullable*/, uint32_t* d_vlen /*nullable*/);
};

// bump allocation inside one scratch buffer, every array on a 256-byte boundary; without a base it only measures
struct Carve {
    uint8_t* base = nullptr;
    uint64_t used = 0;
    template <class T> T* take(uint64_t count)
    {
        T* r = base ? (T*)(base + used) : nullptr;
        used += (sizeof(T) * count + 255) & ~255ull;
        return r;
    }
};
// one scratch area sized and placed by one declaration: lay(c) takes every array from c and assigns the caller's pointers;
// it runs once to measure, `buf` grows to fit (plus 256 bytes of tail), and it runs again to place
template <class Lay> int carve(phant_gpu_ctx* ctx, DevBuf& buf, Lay&& lay)
{
    Carve m;
    lay(m);
    if (int rc = buf.reserve(ctx, m.used + 256)) return rc;
    Carve c{(uint8_t*)buf.ptr};
    lay(c);
    return PHANT_GPU_OK;
}

// a two-phase CUB call: run(temp, bytes) with a null temp only sizes its temporary storage; d_cub grows to fit and run goes
// again for real
template <class Run> int cub_call(phant_gpu_ctx* ctx, Run&& run)
{
    size_t bytes = 0;
    if (cudaError_t e = run((void*)nullptr, bytes)) return ctx->fail(e, "CUB temporary storage size", __FILE__, __LINE__);
    if (int rc = ctx->d_cub.reserve(ctx, bytes)) return rc;
    if (cudaError_t e = run(ctx->d_cub.ptr, bytes)) return ctx->fail(e, "CUB call", __FILE__, __LINE__);
    return PHANT_GPU_OK;
}

// n bytes from the device to dst (nothing when dst is null or n is 0) on the context's stream, counted in d2h_bytes
inline int copy_out(phant_gpu_ctx* ctx, void* dst, const void* src, uint64_t n)
{
    if (!dst || !n) return PHANT_GPU_OK;
    if (cudaError_t e = cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, ctx->stream)) return ctx->fail(e, "cudaMemcpyAsync", __FILE__, __LINE__);
    ctx->stats.d2h_bytes += n;
    return PHANT_GPU_OK;
}
