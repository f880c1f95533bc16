/* phant_gpu.h -- C ABI of libphantgpu.so: phant's trie/hash hot path on NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary (SURVEY.md 8b).  phant has no plugin interface for this path -- `mptize`
 * and `keccak256` are ordinary Zig functions -- so each entry point below names the reference
 * function or hook it stands behind.  Style follows the one C plugin ABI phant already links, EVMC
 * (evmone/evmc/include/evmc/evmc.h:1068-1126: version probe, create/destroy, plain structs).
 * INTEGRATION.md shows the Zig `@cImport` binding and the build.zig lines a maintainer adds.
 *
 * Conventions
 *   - plain C, no exceptions cross the boundary, every size explicit, caller owns every buffer;
 *   - return 0 = OK, negative = error (phant_gpu_strerror).  Accept / reject of a proof is DATA,
 *     never an error code;
 *   - pointers are HOST pointers and the library copies host<->device, unless the context was
 *     switched to device pointers with PHANT_GPU_FLAG_DEVICE_PTRS (benchmarks, callers that already
 *     hold witnesses in HBM).  Device-pointer inputs must be 16-byte aligned and the byte buffers
 *     (msgs / nodes) must be readable for 16 bytes past their last offset.  Host inputs are
 *     validated (monotone offsets, index ranges) before anything is launched; device-pointer inputs
 *     are TRUSTED to be well-formed CSR -- the node CONTENTS are never trusted in either mode.  Device-pointer calls are
 *     ASYNCHRONOUS on the context's stream (its own non-blocking stream unless phant_gpu_set_stream gave it the caller's):
 *     ordering against the caller's own kernels that produce the inputs / consume the outputs is the caller's job --
 *     share the stream, or synchronise on both sides;
 *   - a context owns one device, one stream and its scratch memory; it is not re-entrant: one
 *     context per host thread, or lock around it (phant calls runBlock from httpz worker threads,
 *     src/main.zig:143-149);
 *   - there is NO CPU fallback inside the library: without a usable CUDA device create() fails with
 *     PHANT_GPU_E_NO_DEVICE and the Zig caller keeps its own CPU path.
 */
#ifndef PHANT_GPU_H
#define PHANT_GPU_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PHANT_GPU_ABI_VERSION 2 /* 2: multi-GPU entry points (phant_gpu_comm_*, *_sharded), U kind 1 */

enum {
    PHANT_GPU_OK = 0,
    PHANT_GPU_E_INVALID = -1,   /* bad argument (null pointer, unsorted keys, offsets not monotone ...) */
    PHANT_GPU_E_NO_DEVICE = -2, /* no CUDA device / driver */
    PHANT_GPU_E_OOM = -3,       /* device or pinned-host allocation failed */
    PHANT_GPU_E_CUDA = -4,      /* any other CUDA runtime error (phant_gpu_last_error has the text) */
    PHANT_GPU_E_COMM = -5,      /* NCCL not loadable / communicator missing / a collective failed (phant_gpu_last_error) */
    PHANT_GPU_E_MALFORMED = -6  /* malformed RLP in a *builder* input (never used for proofs) */
};

enum {
    PHANT_GPU_FLAG_DEVICE_PTRS = 1u << 0, /* all data pointers are device pointers; no copies */
    /* Keccak kernel choice (default = staged thread-per-sponge).  See DESIGN.md "Keccak kernels". */
    PHANT_GPU_FLAG_KECCAK_DIRECT = 1u << 4, /* thread-per-sponge, direct global loads */
    PHANT_GPU_FLAG_KECCAK_WARP = 1u << 5,   /* one warp per sponge (north-star layout; slower) */
    PHANT_GPU_FLAG_NO_BINNING = 1u << 6,    /* do not regroup messages by absorb-block count */
    /* chain-form proof batches (node_index == NULL) are hashed and walked by one fused kernel by default; this flag
     * forces the two-kernel path (hash every node, then walk) -- same results, for testing and comparison */
    PHANT_GPU_FLAG_UNFUSED_WALK = 1u << 7
};

typedef struct phant_gpu_ctx phant_gpu_ctx;

typedef struct {
    int32_t device;      /* CUDA device ordinal */
    uint32_t flags;      /* PHANT_GPU_FLAG_* */
    uint64_t reserved[4];
} phant_gpu_config;

/* Environment overrides read by phant_gpu_create: PHANT_GPU_DEVICE (replaces cfg->device), PHANT_GPU_FLAGS (decimal / 0x..,
 * OR-ed into cfg->flags), PHANT_GPU_NCCL_LIB (NCCL library name for the multi-GPU entry points). */
int phant_gpu_abi_version(void);
int phant_gpu_create(phant_gpu_ctx** out, const phant_gpu_config* cfg);
void phant_gpu_destroy(phant_gpu_ctx* ctx);
int phant_gpu_set_flags(phant_gpu_ctx* ctx, uint32_t flags);
/* Run on the caller's CUDA stream (a cudaStream_t passed as void*) instead of the context's own; NULL
 * restores the private stream.  With device pointers every call is then asynchronous on that stream,
 * so the caller can order it against its own kernels / NCCL collectives without a host sync. */
int phant_gpu_set_stream(phant_gpu_ctx* ctx, void* cuda_stream);
const char* phant_gpu_strerror(int code);
const char* phant_gpu_last_error(const phant_gpu_ctx* ctx); /* text of the last CUDA error on this context */

/* Per-call counters, reset by the caller: what bench.py reports as gpu_launches / h2d / d2h and the
 * device time of the dominant kernels (CUDA events on the context's stream). */
typedef struct {
    uint64_t launches;      /* kernels launched by this library */
    uint64_t h2d_bytes, d2h_bytes;
    double keccak_ms;       /* accumulated device time of the batched Keccak kernels (incl. the fused hash-and-walk kernel) */
    double walk_ms;         /* accumulated device time of the proof-walk kernel (fused path: the verdict pass) */
    uint64_t keccak_msgs, keccak_bytes, keccak_perms; /* work the Keccak kernels were given */
    uint64_t reserved[4];
} phant_gpu_stats;
int phant_gpu_get_stats(phant_gpu_ctx* ctx, phant_gpu_stats* out);
int phant_gpu_reset_stats(phant_gpu_ctx* ctx);
int phant_gpu_synchronize(phant_gpu_ctx* ctx);

/* K -- batched Keccak-256.  Replaces hasher.keccak256 (src/crypto/hasher.zig:4-8) for many inputs at
 * once: message i = msgs[off[i] .. off[i+1]) (CSR byte offsets, any alignment, any length incl. 0);
 * out = n*32 digest bytes.  keccak256WithPrefix (hasher.zig:10-17) is the same call on prefix||data. */
int phant_gpu_keccak256_batch(phant_gpu_ctx* ctx, const uint8_t* msgs, const uint64_t* off, uint64_t n, uint8_t* out);
/* The same for DEVICE pointers when the caller knows total_bytes = off[n] - off[0]: nothing is read back, the call is
 * asynchronous on the context's stream (the entry point above needs one host synchronisation to learn the total). */
int phant_gpu_keccak256_batch_async(phant_gpu_ctx* ctx, const uint8_t* msgs, const uint64_t* off, uint64_t n, uint64_t total_bytes, uint8_t* out);

/* M -- == mptize (src/mpt/mpt.zig:38-45).  Keys are byte strings sorted lexicographically (a strict
 * prefix first: KeyVal.lessThan, mpt.zig:31-33), CSR; values CSR.  n == 0 -> empty_mpt_root
 * (mpt.zig:10).  Unsorted or duplicate keys -> PHANT_GPU_E_INVALID (the reference asserts, mpt.zig:39).
 * In device-pointer mode only out_root stays a host pointer. */
int phant_gpu_mpt_root(phant_gpu_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* vals,
                       const uint64_t* val_off, uint64_t n, uint8_t out_root[32]);

/* M (batched) -- many independent tries in one call: trie t holds items [seg_off[t], seg_off[t+1]) of the CSR arrays,
 * each segment sorted like a single mptize input.  All tries are built together as one forest (one set of launches
 * whatever n_tries is): e.g. the transaction / receipt / withdrawal tries (src/blockchain/blockchain.zig:200-203)
 * of a whole range of blocks.  out_roots = n_tries * 32 bytes; an empty segment gives empty_mpt_root. */
int phant_gpu_mpt_roots(phant_gpu_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* vals, const uint64_t* val_off,
                        const uint32_t* seg_off, uint64_t n_tries, uint8_t* out_roots);

/* S -- state root of a flat account table: the body of the missing StateDB.root()
 * (hook: src/blockchain/blockchain.zig:83-85; data model src/state/statedb.zig:16-30,
 * src/state/types.zig:7-33).  Trie contents as in evmone/test/state/mpt_hash.cpp:15-36:
 * key keccak(addr), value rlp([nonce, balance, storage_root, keccak(code)]); storage key
 * keccak(slot), value rlp(trim(value)), zero values skipped (statedb.zig:112-119). */
typedef struct {
    uint64_t n_accounts;
    const uint8_t* addr20;      /* n*20 */
    const uint64_t* nonce;      /* n */
    const uint8_t* balance32;   /* n*32 big endian */
    const uint8_t* code;        /* concatenated code bytes */
    const uint64_t* code_off;   /* n+1 */
    const uint8_t* slot_keys32; /* total_slots*32 */
    const uint8_t* slot_vals32; /* total_slots*32 */
    const uint64_t* slot_off;   /* n+1, in slots */
} phant_gpu_accounts;
int phant_gpu_state_root(phant_gpu_ctx* ctx, const phant_gpu_accounts* accounts, uint8_t out_root[32]);

/* S, sharded across GPUs by the top nibble of keccak(addr) (SURVEY.md 8e): for the accounts handed in, out_roots[v] =
 * hash of the subtree hanging under slot v of the ROOT branch (tries built from key nibble 1 on), bit v of *out_mask set
 * when slot v is populated (unpopulated slots are zero-filled).  Each rank passes the accounts whose top nibble it owns;
 * after one all-gather of 16 x 32 bytes + the masks, every rank hashes the root branch rlp([ref_0 .. ref_15, ""])
 * itself (one K call).  With fewer than two populated slots overall the root is not a branch: the caller falls back to
 * phant_gpu_state_root on the one rank that holds every account.  An account leaf is >= 70 bytes, so a populated slot's
 * reference is always a hash (mpt.zig:104,112 inlining cannot apply). */
int phant_gpu_state_subtree_roots(phant_gpu_ctx* ctx, const phant_gpu_accounts* accounts, uint8_t out_roots[16 * 32], uint32_t* out_mask);

/* V -- batched Merkle-Patricia proof verification: the body of the TODO at
 * src/engine_api/execution_payload.zig:177-178.  Proof p = nodes [proof_first[p], proof_first[p+1]),
 * root first; node j = nodes[node_off[j] .. node_off[j+1]).  n_roots == 1 broadcasts one root.
 * Outputs (each may be NULL): accept_bitmap ceil(n/64) words, bit p = proof p accepted;
 * status[p] 0 reject / 1 present / 2 proven absent; val_off/val_len[p] = slice of `nodes` holding
 * the proven value.  Walk rules: DESIGN.md "Proof walk". */
typedef struct {
    uint64_t n_proofs;
    const uint8_t* nodes;
    const uint64_t* node_off;    /* n_nodes+1 */
    const uint64_t* proof_first; /* n_proofs+1 */
    const uint8_t* keys32;       /* n_proofs*32 */
    const uint8_t* roots32;      /* n_roots*32 */
    uint64_t n_roots;
    uint64_t n_nodes;            /* = proof_first[n_proofs]; may be 0 = "read it from the arrays" (host pointers: */
    uint64_t nodes_bytes;        /* = node_off[n_nodes];      always derived; device pointers: costs a sync)      */
    /* Deduplicated witness (optional): when node_index is not NULL, `nodes` holds every DISTINCT node once
     * (n_nodes of them -- required), each is hashed once, and proof p walks the nodes
     * node_index[proof_first[p] .. proof_first[p+1]).  NULL = chains are contiguous runs of `nodes`. */
    const uint64_t* node_index;
} phant_gpu_proof_batch;
int phant_gpu_verify_proofs(phant_gpu_ctx* ctx, const phant_gpu_proof_batch* in, uint64_t* accept_bitmap,
                            uint8_t* status, uint64_t* val_off, uint32_t* val_len);

/* W -- witness given as an unordered SET of nodes (the shape of an execution witness: `state: [node, ...]`), not as
 * one chain per key.  Every node is hashed once, a device hash table maps digest -> node, and each key is walked
 * from its root resolving every hash reference through the table.  Same node rules as V (R1, R2, R3 without the
 * chain-position clauses); status gets a fourth value: 3 = a node on the key's path is not in the set (incomplete
 * witness).  accept bit = status 1 or 2.  Nodes not on any path are harmless. */
typedef struct {
    uint64_t n_nodes;
    const uint8_t* nodes;
    const uint64_t* node_off; /* n_nodes+1 */
    uint64_t nodes_bytes;     /* = node_off[n_nodes] (device pointers: required; host pointers: derived) */
    uint64_t n_keys;
    const uint8_t* keys32;    /* n_keys*32 */
    const uint8_t* roots32;   /* n_roots*32 */
    uint64_t n_roots;         /* 1 (broadcast) or n_keys */
} phant_gpu_witness;
int phant_gpu_verify_witness(phant_gpu_ctx* ctx, const phant_gpu_witness* in, uint64_t* accept_bitmap, uint8_t* status,
                             uint64_t* val_off, uint32_t* val_len);

/* P -- pre-state reads from an execution witness: what the witness's `state` node set proves about the accounts and storage
 * slots a block touches, decoded, in one call -- the StateDB (src/state/types.zig:13-33) a stateless client fills before it
 * executes the block.  Accounts are walked from roots32 as in W; a present account's body must be one canonical
 * rlp([nonce <= 8 bytes, balance <= 32 bytes, storageRoot 32, codeHash 32]) (no leading zero bytes), else status 0.  Slot i
 * belongs to account slot_account[i] and is walked from that account's decoded storageRoot (which never leaves the device):
 * an absent account makes its slots absent (value 0), a rejected (0) or incomplete (3) account passes its status on to its
 * slots, which are not walked.  A present slot value must be one canonical RLP string of 1..32 bytes with a non-zero first
 * byte, else status 0.  Codes are hashed once and matched to each present account's codeHash: code_index = i with
 * keccak(codes[i]) == codeHash (any such i when codes repeat), PHANT_GPU_CODE_MISSING when none matches,
 * PHANT_GPU_CODE_EMPTY when codeHash == keccak("") or the account is not present.  Outputs use the layout of
 * phant_gpu_accounts (big endian, left padded), so what is read can be handed to phant_gpu_state_root; fields of an account
 * or slot that is not present are zero.  Host pointers: CSR arrays, slot_account < n_accounts and n_roots are checked
 * (PHANT_GPU_E_INVALID, nothing launched).  Device pointers: nodes_bytes / codes_bytes are required, the call is
 * asynchronous, and an out-of-range slot_account gives that slot status 0.  n_nodes, n_codes <= 2^30.  DESIGN.md
 * "P: pre-state reads". */
#define PHANT_GPU_CODE_EMPTY 0xffffffffu   /* codeHash == keccak(""), or the account is not present */
#define PHANT_GPU_CODE_MISSING 0xfffffffeu /* no code in the witness hashes to the account's codeHash */
typedef struct {
    uint64_t n_nodes; const uint8_t* nodes; const uint64_t* node_off; uint64_t nodes_bytes; /* the `state` node set, as W */
    uint64_t n_codes; const uint8_t* codes; const uint64_t* code_off; uint64_t codes_bytes; /* the `codes` (n_codes may be 0) */
    const uint8_t* roots32; uint64_t n_roots;           /* state root: 1 (broadcast) or n_accounts */
    uint64_t n_accounts; const uint8_t* account_keys32; /* keccak(address) */
    uint64_t n_slots; const uint8_t* slot_keys32;       /* keccak(be32(slot)) */
    const uint32_t* slot_account;                       /* n_slots: index into the account list */
} phant_gpu_state_reads;
typedef struct { /* every pointer may be NULL */
    uint8_t* account_status;  /* n_accounts: 0 reject / 1 present / 2 absent / 3 node missing */
    uint64_t* nonce;          /* n_accounts */
    uint8_t* balance32;       /* n_accounts * 32, big endian */
    uint8_t* storage_root32;  /* n_accounts * 32 */
    uint8_t* code_hash32;     /* n_accounts * 32 */
    uint32_t* code_index;     /* n_accounts: index into codes, or PHANT_GPU_CODE_EMPTY / PHANT_GPU_CODE_MISSING */
    uint8_t* slot_status;     /* n_slots: 0 / 1 / 2 / 3 */
    uint8_t* slot_vals32;     /* n_slots * 32, big endian, left padded */
} phant_gpu_state_values;
int phant_gpu_read_state(phant_gpu_ctx* ctx, const phant_gpu_state_reads* in, phant_gpu_state_values* out);

/* B -- logs blooms (row N3 of SURVEY.md 8f): Receipt.calculateLogsBloom / addToBloom
 * (src/types/receipt.zig:37-63) for many receipts at once.  items = the bloom inputs (log addresses 20 B, topics
 * 32 B, ...) CSR; bloom_of_item[i] says which of the n_blooms 2048-bit filters item i belongs to.  Each item is
 * hashed (same batched Keccak kernel) and sets 3 bits: for j in 0..2, bit 0x7ff - (be16(hash[2j..2j+2]) & 0x7ff),
 * most significant bit of byte 0 first.  blooms = n_blooms * 256 bytes (zeroed by the call). */
int phant_gpu_logs_bloom(phant_gpu_ctx* ctx, const uint8_t* items, const uint64_t* item_off, const uint32_t* bloom_of_item,
                         uint64_t n_items, uint64_t n_blooms, uint8_t* blooms);

/* R -- batched sender recovery (row N4 of SURVEY.md 8f): for each i, the secp256k1 public key that signed hashes32[i]
 * under sigs65[i] = r(32, big endian) || s(32) || recid(1), and its address keccak256(X || Y)[12..32] -- the tail of
 * TxSigner.get_sender (src/signer/signer.zig:78-79: ecdsa_signer.erecover, src/crypto/ecdsa.zig:19-21, then
 * hasher.keccak256(pubkey[1..])[12..]).  Decisions are those of libsecp256k1's secp256k1_ecdsa_recover, which the
 * reference calls through zig-eth-secp256k1: ok[i] = 1 and pubkeys65[i] = 0x04 || X || Y, or ok[i] = 0 (r or s zero or
 * >= n, recid > 3, x not on the curve, result at infinity) with zero-filled outputs.  The low-s rule and the EIP-155 `v`
 * decoding are the caller's (signer.zig:41-76, ecdsa.zig:28-36), as in the reference.  pubkeys65 / addresses20 may be
 * NULL.  A failed recovery is data, not an error code. */
int phant_gpu_ecrecover_batch(phant_gpu_ctx* ctx, const uint8_t* hashes32, const uint8_t* sigs65, uint64_t n,
                              uint8_t* pubkeys65, uint8_t* addresses20, uint8_t* ok);

/* U -- resident trie + dirty-frontier root recompute (BASELINE.json "state-root recompute").  Hook: StateDB.root() after
 * a block (src/blockchain/blockchain.zig:83-85).  Two kinds:
 *   kind 0  a complete 16-ary trie with `depth` branch levels (16^depth leaves) whose untouched leaf hashes come from the
 *           synthetic PRNG (the benchmark shape); update rewrites n_dirty leaves at DISTINCT leaf positions (a collision is
 *           refused with PHANT_GPU_E_INVALID and leaves the trie untouched) and re-hashes only the dirty frontier;
 *   kind 1  a SPARSE secure trie over arbitrary 32-byte keys (keccak(address) / keccak(slot)) with arbitrary values, initially
 *           empty: phant_gpu_trie_update is an UPSERT of (key, value) pairs in any order, an empty value DELETES the key
 *           (absent keys are ignored), the same key twice in one call is PHANT_GPU_E_INVALID.  Resident on the device: the
 *           sorted key table, the values, and the references of a dense top of L = floor(log16(n / 16)) nibble levels; an
 *           update re-builds only the buckets (keys sharing an L-nibble prefix) that hold a dirty key -- with all of mptize's
 *           rules: extensions, embedded nodes -- and re-hashes the dirty part of the dense levels.  Host pointers only.
 *           The root always equals mptize over the current key set (src/mpt/mpt.zig:38-45). */
typedef struct phant_gpu_trie phant_gpu_trie;
typedef struct {
    uint32_t kind;  /* 0 = complete synthetic trie, 1 = sparse secure trie */
    uint32_t depth; /* kind 0: branch levels; kind 1: ignored */
    uint64_t seed;
    uint64_t reserved[4];
} phant_gpu_trie_desc;
int phant_gpu_trie_open(phant_gpu_ctx* ctx, const phant_gpu_trie_desc* desc, phant_gpu_trie** out);
int phant_gpu_trie_root(phant_gpu_trie* trie, uint8_t out_root[32]);
int phant_gpu_trie_update(phant_gpu_trie* trie, const uint8_t* keys32, const uint8_t* leaf_vals,
                          const uint32_t* val_off, uint64_t n_dirty, uint8_t out_root[32]);
void phant_gpu_trie_close(phant_gpu_trie* trie);

/* U, world state -- the account trie AND every account's storage trie resident on the device, so that StateDB.root() after a
 * block (src/blockchain/blockchain.zig:83-85) costs what the block changed, storage included.  DESIGN.md §4.3c.
 *   - Keys are hashed by the caller, as for P.  Loading a snapshot is the first apply, with every account in it.
 *   - Each listed account without DELETE is upserted with the nonce, balance and codeHash given; its storage is kept (or
 *     dropped first with CLEAR_STORAGE: a re-created account) and the listed slots are applied to it.  DELETE removes the
 *     account and all of its storage; DELETE on an absent account does nothing.
 *   - A zero slot value deletes the slot (src/state/statedb.zig:112-119); a zero value for an absent slot does nothing.
 *   - The account leaf is rlp([nonce, balance, storageRoot, codeHash]) (evmone mpt_hash.cpp:15-36), as in S: the root always
 *     equals phant_gpu_state_root over the same full state.
 *   - storage_roots32 (nullable, n_accounts * 32) returns the new storage root of each listed account, zero for deleted ones.
 *   - PHANT_GPU_E_INVALID, with the state exactly as it was: the same account key twice; the same (account, slot key) twice;
 *     slot_account out of range; a slot listed for a DELETE account; unknown flag bits; device pointers (host tables only).
 *   - A failure after validation (PHANT_GPU_E_OOM / E_CUDA from a step that runs after the first write) leaves the state
 *     unusable: every later apply and root call returns PHANT_GPU_E_CUDA; close it and load again.
 *   - Device memory stays bounded by the live contents (info.device_bytes).  Not thread safe; one context per state.
 *   - Undo (DESIGN.md §4.3c, "Undo"): with a journal depth > 0 every successful apply, an empty one included, keeps on the device the
 *     record that undoes it (the inverse diff: old nonce, balance, codeHash and slot values of what it listed), so that a
 *     block whose root does not match its header, or the blocks a reorg leaves, can be taken back without a reload.  A refused
 *     apply records nothing.  The record is reserved before the apply's first write: if that fails the apply is refused
 *     (PHANT_GPU_E_OOM) with the state exactly as it was.  Depth 0, the default, keeps no records. */
typedef struct phant_gpu_resident_state phant_gpu_resident_state;
#define PHANT_GPU_ACCOUNT_DELETE 1u        /* remove the account and all of its storage */
#define PHANT_GPU_ACCOUNT_CLEAR_STORAGE 2u /* drop its storage before this diff's slots are applied (re-created account) */
typedef struct {
    uint64_t n_accounts;
    const uint8_t* account_keys32; /* keccak(address), n * 32 */
    const uint8_t* account_flags;  /* n, PHANT_GPU_ACCOUNT_*; NULL = all 0 */
    const uint64_t* nonce;         /* n */
    const uint8_t* balance32;      /* n * 32 big endian */
    const uint8_t* code_hash32;    /* n * 32 */
    uint64_t n_slots;
    const uint32_t* slot_account;  /* n_slots: index into the account list above */
    const uint8_t* slot_keys32;    /* keccak(be32(slot)) */
    const uint8_t* slot_vals32;    /* 32 bytes big endian; all zero = delete */
} phant_gpu_state_diff;
typedef struct {
    uint64_t n_accounts, n_slots, device_bytes; /* device_bytes includes the journal */
    uint64_t journal_applies;                   /* how many applies revert can undo */
    uint64_t journal_bytes;                     /* device memory of the undo journal */
    uint64_t reserved[2];
} phant_gpu_state_info; /* a type of its own name: C shares one namespace between typedefs and functions */
int phant_gpu_resident_state_open(phant_gpu_ctx* ctx, phant_gpu_resident_state** out); /* empty: root = keccak(0x80) */
int phant_gpu_resident_state_apply(phant_gpu_resident_state* st, const phant_gpu_state_diff* diff, uint8_t out_root[32],
                                   uint8_t* storage_roots32);
int phant_gpu_resident_state_root(phant_gpu_resident_state* st, uint8_t out_root[32]);
int phant_gpu_resident_state_info(phant_gpu_resident_state* st, phant_gpu_state_info* out);
/* Keep the undo records of the last `depth` successful applies on the device (0 = none, the default: apply behaves exactly as
 * before).  A smaller depth drops the oldest records; depth > 1024 -> PHANT_GPU_E_INVALID. */
int phant_gpu_resident_state_set_journal(phant_gpu_resident_state* st, uint32_t depth);
/* Undo the last n_applies successful applies, newest first; out_root = the root before the oldest of them.  n_applies == 0
 * returns the current root.  More than the journal holds -> PHANT_GPU_E_INVALID, nothing changes.  Undone records are consumed.
 * No diff data crosses PCIe: each record is replayed on the device, and the root after it must equal the root the record saved
 * (a mismatch, or a failure after a replay's first write, leaves the state unusable as for apply; a failure before it leaves
 * the records already undone undone).  On an unusable state, set_journal and revert return PHANT_GPU_E_CUDA. */
int phant_gpu_resident_state_revert(phant_gpu_resident_state* st, uint32_t n_applies, uint8_t out_root[32]);
/* The execution witness of a block, from the state as it is now (before the block): the trie nodes of the pre-state that `diff`
 * (as for apply) reads or changes.  The state is not changed: root, info's tables and journal, and everything resident stay as
 * they were, and a failure leaves the state usable.  The node set holds, each node once (distinct bytes, across tries too),
 * ordered by keccak digest:
 *   - for every listed account key, its path in the account trie (from the root to its leaf, or to the node where its path
 *     leaves the trie); for every DELETE account, the paths of the nearest account keys before and after it that the diff does
 *     not DELETE, where they exist;
 *   - for every listed slot of an account present before the block, listed without DELETE or CLEAR_STORAGE and with storage:
 *     its path in that storage trie, and for a zero write the paths of the nearest slot keys of the account before and after
 *     it that the diff does not zero.
 * A trie's root is always included, other nodes only when their encoding is 32 bytes or more (embedded nodes travel inside their
 * parents).  The set holds every node phant_gpu_transition_roots needs for this diff from this state's root.  Every refusal of
 * apply is a refusal here (PHANT_GPU_E_INVALID, nothing held); on an unusable state PHANT_GPU_E_CUDA.  The result stays on the
 * device (counted in info's device_bytes) until witness_copy or the next witness, apply, set_journal, revert or close. */
typedef struct {
    uint64_t n_nodes, nodes_bytes;
    uint64_t reserved[2];
} phant_gpu_witness_size;
int phant_gpu_resident_state_witness(phant_gpu_resident_state* st, const phant_gpu_state_diff* diff, phant_gpu_witness_size* out);
/* Copy the result of the last witness call to host memory and release it: nodes = nodes_bytes bytes, node_off = n_nodes + 1
 * offsets.  Nothing held -> PHANT_GPU_E_INVALID. */
int phant_gpu_resident_state_witness_copy(phant_gpu_resident_state* st, uint8_t* nodes, uint64_t* node_off);
void phant_gpu_resident_state_close(phant_gpu_resident_state* st);

/* T -- state transition roots: the post-state root of each of n_blocks blocks, from the witness's `state` node set, the block's
 * parent state root and what execution wrote -- the root a stateless client compares with the header (hook:
 * src/blockchain/blockchain.zig:83-85; StatelessPayloadStatusV1.state_root, src/engine_api/execution_payload.zig:20-25).
 * DESIGN.md "T: state transition roots".
 *   - The diff means, per block, what it means for phant_gpu_resident_state_apply (hashed keys; full nonce, balance and codeHash
 *     per upsert; CLEAR_STORAGE drops the old storage first; DELETE removes the account and its storage; a zero slot value
 *     deletes the slot; deleting something absent does nothing).  Account i belongs to block account_block[i] (NULL: block 0).
 *   - Blocks are independent: each is applied to its own pre_roots32[b]; an account may be listed in several blocks, and
 *     blocks share the one node set (nodes are found by hash).
 *   - status[b] = 1: post_roots32[b] is the block's post-state root.  0: a node the computation reads breaks R2-R4 (DESIGN.md
 *     "Proof walk"; every item of such a node is checked), a leaf's key is not 64 nibbles, or a listed present account's body
 *     does not decode as for P.  3: a node the computation needs is not in the set.  post_roots32[b] is zero unless status is
 *     1; storage_roots32 (nullable, n_accounts * 32) holds each listed account's new storage root, zero for DELETE accounts and
 *     for blocks whose status is not 1.  An insufficient witness is data, not an error code.
 *   - The set must hold: the pre-state path of every listed account key under its block's pre-root; the pre-state path of every
 *     listed slot key under its account's pre-state storage root (not for accounts absent before the block, nor for accounts
 *     listed with DELETE or CLEAR_STORAGE); and, for every branch the diff leaves with a single child, that child when the
 *     branch references it by hash.  Nothing else: an insert that splits an extension does not need the node below it.  This
 *     is what a geth-style witness holds (the nodes read, plus the child resolved when a branch collapses).
 *   - The call never returns status 1 with a root that differs from the true post-state root.
 *   - PHANT_GPU_E_INVALID, nothing written: the same account key twice in one block; the same (account, slot key) twice;
 *     slot_account out of range; a slot of a DELETE account; unknown flag bits; account_block[i] >= n_blocks; n_blocks == 0;
 *     device pointers (host pointers only).  n_nodes <= 2^30. */
typedef struct {
    uint64_t n_nodes; const uint8_t* nodes; const uint64_t* node_off; uint64_t nodes_bytes; /* union of the blocks' `state` node sets, as W */
    uint64_t n_blocks;
    const uint8_t* pre_roots32;    /* n_blocks * 32: each block's parent state root */
    const uint32_t* account_block; /* diff->n_accounts: the block each listed account belongs to; NULL = all in block 0 */
} phant_gpu_transition;
int phant_gpu_transition_roots(phant_gpu_ctx* ctx, const phant_gpu_transition* in, const phant_gpu_state_diff* diff,
                               uint8_t* post_roots32 /* n_blocks * 32 */, uint8_t* status /* n_blocks */,
                               uint8_t* storage_roots32 /* nullable, diff->n_accounts * 32 */);

/* ---- multi-GPU (SURVEY.md 8e): proofs shard by contiguous index range, one context per GPU, the only exchange is the
 * accept bitmap.  The reference runs block processing on httpz worker threads (src/main.zig:143-149): either one process
 * with one context + host thread per GPU (phant_gpu_comm_init_local), or one process per GPU (phant_gpu_comm_init with an
 * id from rank 0, carried by whatever channel the host has).  NCCL is loaded at run time (libnccl.so.2, override with
 * PHANT_GPU_NCCL_LIB); single-GPU users never touch it.  Failures return PHANT_GPU_E_COMM. ---- */
#define PHANT_GPU_COMM_ID_BYTES 128
int phant_gpu_comm_get_unique_id(uint8_t id[PHANT_GPU_COMM_ID_BYTES]);                            /* rank 0, then distribute */
int phant_gpu_comm_init(phant_gpu_ctx* ctx, const uint8_t id[PHANT_GPU_COMM_ID_BYTES], int rank, int world); /* collective */
int phant_gpu_comm_init_local(phant_gpu_ctx** ctxs, int n); /* one process: n contexts on n devices, rank i = ctxs[i]; afterwards
                                                               drive each context from its own host thread */
int phant_gpu_comm_info(const phant_gpu_ctx* ctx, int* rank, int* world, int* nccl_version);
/* Optional PEER TRANSPORT for the gathered accept bitmap (same node, NVLink): a collective call that maps one small symmetric
 * region of every rank into every other rank (cudaIpc; one process per GPU -- contexts that share a process keep NCCL).  Afterwards
 * device-pointer calls of phant_gpu_verify_proofs_sharded with equal, 64-aligned shards of at most max_n_global proofs need
 * no collective launch: the walk kernel's epilogue stores each ballot word straight into every rank's gathered bitmap and
 * publishes the step, and the comm stream only waits for the peers' words and copies the bitmap out.  Everything else keeps
 * using NCCL.  PHANT_GPU_E_COMM when a mapping is not possible on some rank: nothing changes, NCCL stays in use.  A rank
 * that stops answering makes the waiting kernels give up after 4 s; phant_gpu_comm_peer_status reports it. */
int phant_gpu_comm_enable_peer(phant_gpu_ctx* ctx, uint64_t max_n_global);
int phant_gpu_comm_disable_peer(phant_gpu_ctx* ctx); /* collective: unmap, back to the NCCL gather */
int phant_gpu_comm_peer_status(phant_gpu_ctx* ctx, int* enabled, uint64_t* steps, int* timed_out);
int phant_gpu_comm_fence(phant_gpu_ctx* ctx);   /* the context's stream waits (on the device) for every collective issued so far */
int phant_gpu_comm_destroy(phant_gpu_ctx* ctx); /* also done by phant_gpu_destroy */
/* Rank r of `world` owns proofs [lo, hi): contiguous, every boundary but the last a multiple of 64 so that bitmap words
 * are disjoint.  A gathered bitmap has phant_gpu_sharded_bitmap_words(n, world) words (>= ceil(n/64): equal slices). */
int phant_gpu_shard_range(uint64_t n, int rank, int world, uint64_t* lo, uint64_t* hi);
uint64_t phant_gpu_sharded_bitmap_words(uint64_t n, int world);
/* V across GPUs: `local` holds THIS rank's shard of a batch of n_global proofs (local->n_proofs == hi - lo); on return
 * global_bitmap holds every rank's accept bits (bit p = proof p of the global batch); status / val_* cover the local shard.
 * Host pointers: synchronous.  Device pointers: Keccak + walk are enqueued on the context's stream and ONE ncclAllGather on
 * the context's comm stream behind an event -- the next call's Keccak overlaps it; the walk that next writes the same
 * global_bitmap buffer waits for it on the device (alternate two buffers and nothing ever waits); phant_gpu_comm_fence or
 * phant_gpu_synchronize before reading. */
int phant_gpu_verify_proofs_sharded(phant_gpu_ctx* ctx, const phant_gpu_proof_batch* local, uint64_t n_global,
                                    uint64_t* global_bitmap, uint8_t* status, uint64_t* val_off, uint32_t* val_len);
/* Per-block verdicts when BLOCKS are sharded (BASELINE.json "1000 blocks x 300 tx"): counts[b] = proofs of block b that
 * were not accepted (status 0 or 3), summed over ranks with one all-reduce; block b is valid iff counts[b] == 0. */
int phant_gpu_block_reject_counts(phant_gpu_ctx* ctx, const uint8_t* status, const uint32_t* block_of_proof, uint64_t n_proofs,
                                  uint64_t n_blocks, uint32_t* counts);
/* S across GPUs: rank r passes the accounts whose top nibble of keccak(address) it owns (phant_gpu_nibble_owner: contiguous
 * slot ranges); subtree roots are built locally, ONE all-gather of 528 bytes per rank follows and every rank hashes the
 * root branch itself.  Fewer than two populated slots overall: the one rank holding accounts computes the plain root and
 * broadcasts it.  Host pointers only. */
int phant_gpu_nibble_owner(int nibble, int world);
int phant_gpu_state_root_sharded(phant_gpu_ctx* ctx, const phant_gpu_accounts* mine, uint8_t out_root[32]);

/* Synthetic witnesses generated on the device (SURVEY.md 8d; byte-identical to oracle/synth.c).
 * All pointers are DEVICE pointers regardless of the context flags.  which: 2 = account proofs of
 * `depth` nodes (config C2), 3 = storage proofs depth 4..12 (config C3; depth ignored).
 * phant_gpu_synth_sizes fills host totals so the caller can allocate. */
int phant_gpu_synth_sizes(phant_gpu_ctx* ctx, int which, uint64_t seed, uint64_t first_index, uint64_t n,
                          uint32_t depth, uint64_t* total_nodes, uint64_t* total_bytes);
int phant_gpu_synth(phant_gpu_ctx* ctx, int which, uint64_t seed, uint64_t first_index, uint64_t n, uint32_t depth,
                    int corrupt, uint8_t* nodes, uint64_t* node_off, uint64_t* proof_first, uint8_t* keys32,
                    uint8_t* roots32);

#ifdef __cplusplus
}
#endif
#endif /* PHANT_GPU_H */
