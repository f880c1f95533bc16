// common.cuh -- declarations shared by the translation units of libphantgpu.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace phant {

enum KeccakVariant { KECCAK_STAGED = 0, KECCAK_DIRECT = 1, KECCAK_WARP = 2 };

// abi.cu: a host CSR's offsets must start at off[0] (any value) and be monotone; returns the last offset via *total
int check_offsets_host(const uint64_t* off, uint64_t n, uint64_t* total);

// keccak_kernels.cu
int keccak_num_sms(int device);
cudaError_t launch_keccak(cudaStream_t s, int device, KeccakVariant variant, const uint8_t* msgs, const uint64_t* off,
                          const uint32_t* order, uint64_t n, uint8_t* out, uint32_t* summary /*nullable*/,
                          const uint64_t* len = nullptr /*nullable: message m = msgs[off[m] .. off[m] + len[m])*/);
// regrouping by permutation count (stable 16-bucket counting sort, two launches): classify fills hist[blocks][16], counts the
// permutations and leaves global start positions in hist; regroup writes `order`
uint64_t keccak_regroup_scratch_bytes(int device, uint64_t n);
// proofs = true: the same sort over chain-form proofs (`off` = proof_first) by node count, without permutation statistics
cudaError_t launch_keccak_classify(cudaStream_t s, int device, const uint64_t* off, uint64_t n, uint32_t* hist, uint32_t* ticket,
                                   unsigned long long* perms, bool proofs = false);
cudaError_t launch_keccak_regroup(cudaStream_t s, int device, const uint64_t* off, uint64_t n, const uint32_t* start, uint32_t* order,
                                  bool proofs = false);
// fused hash-and-walk of chain-form proofs (node_index == NULL; `nodes` 16-byte aligned): status / value slice per proof,
// permutations of all nodes added to *perms; proof order through `order` (nullable)
cudaError_t launch_verify_fused(cudaStream_t s, int device, const uint8_t* nodes, const uint64_t* node_off, const uint64_t* proof_first,
                                const uint32_t* order, uint64_t n, const uint8_t* keys32, const uint8_t* roots32, uint64_t n_roots,
                                uint8_t* status, uint64_t* val_off /*nullable*/, uint32_t* val_len /*nullable*/, unsigned long long* perms);

// Peer-memory epilogue of the proof walk (comm.cu "peer transport"): every warp stores its ballot word straight into the
// gathered bitmap of EVERY rank of the node through NVLink peer mappings (lane r < world stores to rank r: one predicated
// store instruction), and the last CTA to finish publishes "step s of rank `me` has landed" in every rank's flag array.
constexpr int PEER_MAX_WORLD = 16;
struct PeerOut {
    uint32_t* dst[PEER_MAX_WORLD];         // rank r's bitmap of this step's buffer, at THIS rank's slice (32-bit words)
    unsigned long long* ready[PEER_MAX_WORLD]; // in rank r's region: ready[buffer][me]
    const unsigned long long* done;        // in MY region: done[buffer][0..world): rank r has copied step (value) out of this buffer
    unsigned long long wait_done;          // wait until done[r] >= this for every r before touching remote memory (0 = no wait)
    unsigned long long step;               // value to publish
    uint32_t* ticket;                      // CTA counter (device memory of this rank)
    uint32_t* err;                         // set to 1 when a wait times out
    uint32_t world;
};

// walk_kernel.cu
cudaError_t launch_walk(cudaStream_t s, int device, uint64_t n_proofs, const uint8_t* nodes, const uint64_t* node_off,
                        const uint64_t* node_index /*nullable*/, const uint64_t* proof_first, const uint8_t* keys32, const uint8_t* roots32, uint64_t n_roots,
                        const uint8_t* digests, const uint32_t* summary /*nullable*/, uint64_t* bitmap, uint8_t* status,
                        uint64_t* val_off, uint32_t* val_len, const PeerOut* peer = nullptr /*nullable: fused gather over peer memory*/);

// accept words from per-proof status (PRESENT or ABSENT = accept): bitmap words [0, ceil(n / 64)) are all written
cudaError_t launch_verdict(cudaStream_t s, int device, const uint8_t* status, uint64_t n, uint64_t* bitmap);

cudaError_t launch_peer_collect(cudaStream_t s, const unsigned long long* ready, uint32_t world, unsigned long long step, const void* src, void* dst,
                                uint64_t bytes, const PeerOut& sig);

cudaError_t launch_bag_build(cudaStream_t s, int device, const uint8_t* digests, uint64_t n_nodes, uint32_t* table, uint32_t capacity);
cudaError_t launch_walk_bag(cudaStream_t s, int device, uint64_t n_keys, const uint8_t* nodes, const uint64_t* node_off, const uint8_t* keys32,
                            const uint8_t* roots32, uint64_t n_roots, const uint8_t* digests, const uint32_t* summary, const uint32_t* table,
                            uint32_t capacity, uint64_t* bitmap, uint8_t* status, uint64_t* val_off, uint32_t* val_len);

// state_read.cu: pre-state reads (entry point P).  The account pass writes a record per account (status byte + decoded
// storage root, 32-byte aligned) that the slot pass gathers; every output pointer is nullable.
struct StateOut {
    uint8_t* account_status;
    uint64_t* nonce;
    uint8_t* balance32;
    uint8_t* storage_root32;
    uint8_t* code_hash32;
    uint32_t* code_index;
    uint8_t* slot_status;
    uint8_t* slot_vals32;
};
cudaError_t launch_read_accounts(cudaStream_t s, int device, uint64_t n_accounts, const uint8_t* nodes, const uint64_t* node_off,
                                 const uint8_t* digests, const uint32_t* summary, const uint32_t* table, uint32_t capacity,
                                 const uint8_t* keys32, const uint8_t* roots32, uint64_t n_roots, const uint8_t* code_digests,
                                 const uint32_t* code_table /*nullable: no codes*/, uint32_t code_capacity, uint8_t* rec_roots32,
                                 uint8_t* rec_status, const StateOut& out);
cudaError_t launch_read_slots(cudaStream_t s, int device, uint64_t n_slots, const uint8_t* nodes, const uint64_t* node_off,
                              const uint8_t* digests, const uint32_t* summary, const uint32_t* table, uint32_t capacity,
                              const uint8_t* keys32, const uint32_t* slot_account, uint64_t n_accounts, const uint8_t* rec_roots32,
                              const uint8_t* rec_status, const StateOut& out);

// synth.cu
cudaError_t launch_synth_c2(cudaStream_t s, int device, uint64_t seed, uint64_t first_index, uint64_t n, uint32_t depth,
                            int corrupt, uint8_t* nodes, uint64_t* node_off, uint64_t* proof_first, uint8_t* keys32,
                            uint8_t* roots32);
cudaError_t launch_synth_c3_sizes(cudaStream_t s, int device, uint64_t seed, uint64_t first_index, uint64_t n,
                                  uint64_t* n_nodes_per, uint64_t* n_bytes_per);
cudaError_t launch_synth_c3(cudaStream_t s, int device, uint64_t seed, uint64_t first_index, uint64_t n, int corrupt,
                            const uint64_t* node_first /* exclusive scan of nodes per proof, n+1 */,
                            const uint64_t* byte_first /* exclusive scan of bytes per proof, n+1 */, uint8_t* nodes,
                            uint64_t* node_off, uint8_t* keys32, uint8_t* roots32);

} // namespace phant
