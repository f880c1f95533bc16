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
    DevBuf d_first, d_keys, d_roots, d_digests, d_bitmap, d_status, d_voff, d_vlen, d_summary, d_index; // V
    DevBuf d_cls, d_cls2, d_idx, d_order, d_cub, d_perms;                 // regrouping
    DevBuf d_tmp_a, d_tmp_b, d_scan_a, d_scan_b;                          // synth / builders
    DevBuf d_b0, d_b1, d_b2, d_b3, d_b4, d_b5, d_b6, d_b7, d_b8, d_b9;    // trie builder scratch
    DevBuf st_in, st_hash, st_seg, st_tmp, st_sort, st_acc;               // state-root staging
    DevBuf sr_in, sr_out, sr_rec, sr_code;                                // pre-state reads: staging, outputs, account records, code table
    DevBuf tr_in, tr_keys, tr_sort, tr_front[2], tr_items, tr_work, tr_vals;  // transition roots (trie.cu "T")
    bool perms_init = false, perms_pending = false;

    std::array<DevBuf*, 53> all_bufs()
    {
        return {&d_msgs, &d_off, &d_out, &d_first, &d_keys, &d_roots, &d_digests, &d_bitmap, &d_status, &d_voff, &d_vlen,
                &d_cls, &d_cls2, &d_idx, &d_order, &d_cub, &d_perms, &d_tmp_a, &d_tmp_b, &d_scan_a, &d_scan_b,
                &d_b0, &d_b1, &d_b2, &d_b3, &d_b4, &d_b5, &d_b6, &d_b7, &d_b8, &d_b9,
                &st_in, &st_hash, &st_seg, &st_tmp, &st_sort, &st_acc, &d_summary, &d_index, &d_comm, &d_rej,
                &sr_in, &sr_out, &sr_rec, &sr_code, &tr_in, &tr_keys, &tr_sort, &tr_front[0], &tr_front[1], &tr_items, &tr_work, &tr_vals};
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
    // messages in slots: message m = d_msgs[d_off[m] .. d_off[m] + d_len[m]); no regrouping, no statistics pass
    int hash_slots(const uint8_t* d_msgs, const uint64_t* d_off, const uint64_t* d_len, uint64_t n, uint8_t* d_out);
    // chain-form proofs (no node_index) in one fused hash-and-walk kernel, then the verdict pass (abi.cu); fused_ok() says
    // whether this call may take that path
    bool fused_ok(const uint8_t* d_nodes, uint64_t n_proofs, uint64_t n_nodes) const;
    int verify_fused(const uint8_t* d_nodes, const uint64_t* d_node_off, uint64_t n_nodes, uint64_t total_bytes, const uint64_t* d_proof_first,
                     uint64_t n_proofs, const uint8_t* d_keys, const uint8_t* d_roots, uint64_t n_roots, uint64_t* d_bitmap /*nullable*/,
                     uint8_t* d_status /*nullable*/, uint64_t* d_voff /*nullable*/, uint32_t* d_vlen /*nullable*/);
    // trie.cu
    int build_forest(const uint8_t* d_keys, const uint32_t* d_key_off, const uint8_t* d_vals, const uint64_t* d_val_off, uint32_t n,
                     const uint32_t* d_seg_off, uint32_t n_seg, const uint32_t* d_seg_of_key, uint8_t* d_roots,
                     int slots_hint = 0 /* > 0: slot layout with this leaf stride; < 0: decide on the device; 0: general layout */,
                     uint32_t start_depth = 0 /* key nibbles consumed above every segment's root */,
                     const uint8_t* d_leaf_cache = nullptr /* n x 33: leaf references of an earlier build (resident tries), see trie.cu */,
                     uint8_t* d_leaf_cache_out = nullptr /* n x 33: the references of this build */,
                     const uint32_t* d_seg_start = nullptr /* n_seg: start_depth per segment (nullable: start_depth for all) */,
                     const struct ForestExport* xp = nullptr /* nullable: copy out the nodes on given key paths (trie.cu) */);
    int sort_by_segment_and_hash(const uint8_t* d_hashes, const uint32_t* d_seg, uint32_t n, uint32_t* d_perm_out, DevBuf& scratch);
};
