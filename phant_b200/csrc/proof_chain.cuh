// proof_chain.cuh -- one key's proof chain over a node set sorted by digest (phant_gpu_resident_state_prove in
// include/phant_gpu.h): from the trie's root, find each node referenced by hash by binary search over the digests, decode it
// with the transition roots' node decoder and follow the key's nibbles, walking embedded children in place.  Per thread,
// device code, called by the prove kernels in trie.cu.  pc_node_at walks the same way by nibble path for the trie-node
// kernels (phant_gpu_resident_state_trie_nodes, DESIGN.md §4.3k).
//
// Kept in a header of its own, like transition.cuh, so that the same statements can be compiled as HOST code by the test
// harness (tests/hostcheck/proof_chain_host.cpp) and compared with the CPU trie's proofs (oracle_trie_prove) on a machine
// without a GPU.  DESIGN.md §4.3f.
#pragma once
#include <stdint.h>

#include "transition.cuh" // tn_decode, tn_path_nibble, tk_nibble

namespace phant {
namespace {

enum { PC_BAD = 0, PC_PRESENT = 1, PC_ABSENT = 2 };

// The node set: node k is bytes[off[k] .. off[k+1]) and its keccak digest is dig[32k .. 32k+32); digests strictly increase.
struct PcSet {
    const uint8_t* bytes;
    const uint64_t* off;
    const uint8_t* dig;
    uint32_t n;
};
// A walk's result: status, chain length, and for a present key the payload of its leaf's value item (bytes + val_off).
struct PcWalk {
    uint32_t status, len;
    uint64_t val_off;
    uint32_t val_len;
};

__device__ __forceinline__ int pc_cmp32(const uint8_t* a, const uint8_t* b)
{
    for (int i = 0; i < 32; ++i)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
// the node whose digest is `ref`, or s.n
__device__ __forceinline__ uint32_t pc_find(const PcSet& s, const uint8_t* ref)
{
    uint32_t a = 0, b = s.n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (pc_cmp32(s.dig + 32ull * mid, ref) < 0) a = mid + 1; else b = mid;
    }
    return a < s.n && pc_cmp32(s.dig + 32ull * a, ref) == 0 ? a : s.n;
}

// The chain of `key` (64 nibbles) under `root`: the root node, then every node its lookup path references by hash (the nodes
// of 32 bytes or more), root first; an embedded node is walked inside its parent and adds no entry.  The walk stops at the
// key's leaf (present) or where the key's path leaves the trie (absent): an empty branch child, or an extension or leaf path
// that differs from the key's nibbles.  A root equal to `empty_root` is the empty trie: an empty chain, absent.
// chain (nullable) receives the node indices.  PC_BAD: a referenced node is not in the set or breaks the node rules.
__device__ PcWalk pc_walk(const PcSet& s, const uint8_t* root, const uint8_t* empty_root, const uint8_t* key, uint64_t* chain)
{
    PcWalk w{PC_ABSENT, 0, 0, 0};
    if (pc_cmp32(root, empty_root) == 0) return w;
    const uint8_t* ref = root; // the next node by its digest; nullptr: `node` is an embedded child, already in hand
    const uint8_t* node = nullptr;
    uint32_t len = 0, d = 0;
    for (;;) {
        if (ref) {
            const uint32_t k = pc_find(s, ref);
            if (k == s.n) { w.status = PC_BAD; return w; }
            if (chain) chain[w.len] = k;
            ++w.len;
            node = s.bytes + s.off[k];
            len = (uint32_t)(s.off[k + 1] - s.off[k]);
        }
        TNode t;
        if (!tn_decode(node, len, t)) { w.status = PC_BAD; return w; }
        uint32_t c = 0; // the child the key follows
        if (t.kind == TN_BRANCH) {
            if (d >= 64) { w.status = PC_BAD; return w; } // a secure trie's keys end in leaves
            c = tk_nibble(key, d++);
        } else {
            if (d + t.plen > 64) return w;
            for (uint32_t j = 0; j < t.plen; ++j)
                if (tn_path_nibble(node, t, j) != tk_nibble(key, d + j)) return w;
            d += t.plen;
            if (t.kind == TN_LEAF) {
                if (d != 64) return w;
                w.status = PC_PRESENT;
                w.val_off = (uint64_t)(node - s.bytes) + t.val_off;
                w.val_len = t.val_len;
                return w;
            }
        }
        if (t.c_kind[c] == TC_EMPTY) return w;
        if (t.c_kind[c] == TC_HASH) {
            ref = node + t.c_off[c];
            continue;
        }
        node += t.c_off[c];
        len = t.c_len[c];
        ref = nullptr;
    }
}

// The node that starts at nibble path `path` (its first plen <= 64 nibbles, tk_nibble order) under `root`
// (phant_gpu_resident_state_trie_nodes): PC_PRESENT and its index in the set when that node is the root or is referenced by
// hash; PC_ABSENT when the trie is empty, the path leaves the trie (an empty branch child, an extension path that differs),
// ends inside an extension's or a leaf's path or below a leaf, or the node there is embedded in its parent.  The walk follows
// the path as pc_walk follows a key and stops once plen nibbles are consumed.  PC_BAD: a referenced node is not in the set or
// breaks the node rules.
struct PcAt {
    uint32_t status, index;
};
__device__ PcAt pc_node_at(const PcSet& s, const uint8_t* root, const uint8_t* empty_root, const uint8_t* path, uint32_t plen)
{
    PcAt a{PC_ABSENT, 0};
    if (pc_cmp32(root, empty_root) == 0) return a;
    const uint8_t* ref = root; // as in pc_walk
    const uint8_t* node = nullptr;
    uint32_t len = 0, d = 0, k = 0;
    for (;;) {
        if (ref) {
            k = pc_find(s, ref);
            if (k == s.n) { a.status = PC_BAD; return a; }
            node = s.bytes + s.off[k];
            len = (uint32_t)(s.off[k + 1] - s.off[k]);
        }
        if (d == plen) {
            if (ref) { a.status = PC_PRESENT; a.index = k; }
            return a;
        }
        TNode t;
        if (!tn_decode(node, len, t)) { a.status = PC_BAD; return a; }
        uint32_t c = 0;
        if (t.kind == TN_BRANCH) {
            c = tk_nibble(path, d++);
        } else {
            if (t.kind == TN_LEAF || d + t.plen > plen) return a;
            for (uint32_t j = 0; j < t.plen; ++j)
                if (tn_path_nibble(node, t, j) != tk_nibble(path, d + j)) return a;
            d += t.plen;
        }
        if (t.c_kind[c] == TC_EMPTY) return a;
        if (t.c_kind[c] == TC_HASH) {
            ref = node + t.c_off[c];
            continue;
        }
        node += t.c_off[c];
        len = t.c_len[c];
        ref = nullptr;
    }
}

} // namespace
} // namespace phant
