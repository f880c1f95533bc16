// transition.cuh -- one node of the state-transition root (entry point T of include/phant_gpu.h): decode it and split the sorted
// diff keys that lie under it among its children.  Per thread, device code, called by the T kernels in trie.cu.
//
// Kept in a header of its own, like walk_one.cuh and state_read.cuh, so that the same statements can be compiled as HOST code
// by the test harness (tests/hostcheck/transition_host.cpp) and compared with the CPU statement tests/transition_oracle.py on a
// machine without a GPU.  Rules: DESIGN.md "T: state transition roots".
#pragma once
#include <stdint.h>

#include "walk_one.cuh" // Item / rlp_item: the canonical-RLP rules of the walk

namespace phant {
namespace {

enum { TN_BAD = 0, TN_LEAF = 1, TN_EXT = 2, TN_BRANCH = 3 };
enum { TC_EMPTY = 0, TC_HASH = 1, TC_EMBED = 2 };

// A decoded node.  Offsets are from the node's first byte.
struct TNode {
    uint32_t kind;
    uint32_t path_off, plen, odd; // leaf / extension: the hex-prefix bytes, the path's nibble count, its odd flag
    uint32_t val_off, val_len;    // leaf: the value's payload
    uint32_t c_off[16], c_len[16]; // extension: child 0; branch: children 0..15.  TC_HASH: the 32 digest bytes; TC_EMBED: the node
    uint8_t c_kind[16];
};

__device__ __forceinline__ uint32_t tn_path_nibble(const uint8_t* node, const TNode& t, uint32_t j)
{
    const uint32_t q = j + 2 - t.odd; // nibble index inside the hex-prefix bytes (the flag nibble is 0, an even path's pad is 1)
    const uint8_t b = node[t.path_off + (q >> 1)];
    return (q & 1) ? (b & 15u) : (b >> 4);
}

// a child reference: the empty string, a 32-byte hash, or an embedded node (an RLP list shorter than 32 bytes)
__device__ __forceinline__ bool tn_child(const Item& it, uint32_t off, uint8_t& kind, uint32_t& c_off, uint32_t& c_len)
{
    if (it.is_list) {
        const uint32_t tot = it.pay_off + it.pay_len;
        if (tot >= 32) return false;
        kind = TC_EMBED; c_off = off; c_len = tot;
        return true;
    }
    if (it.pay_len == 0) { kind = TC_EMPTY; c_off = off; c_len = 0; return true; }
    if (it.pay_len != 32) return false;
    kind = TC_HASH; c_off = off + it.pay_off; c_len = 32;
    return true;
}

// R2-R4 for every item of the node, not only the one a key selects: one canonical RLP list of 17 or 2 items and nothing after
// it; a branch holds 16 child references and an empty value (every key of a secure trie has 64 nibbles); a leaf or extension
// starts with a hex-prefix path (flag <= 3, zero pad nibble when even, at most 64 nibbles); a leaf value is a string; an
// extension has a non-empty path and a non-empty child.
__device__ bool tn_decode(const uint8_t* node, uint32_t len, TNode& t)
{
    t.kind = TN_BAD;
    Item top;
    const uint32_t tot = rlp_item(node, len, top);
    if (tot == 0 || !top.is_list || tot != len) return false;
    const uint32_t end = top.pay_off + top.pay_len;
    Item i0{}, i1{};
    uint32_t o0 = 0, o1 = 0, cnt = 0;
    for (uint32_t o = top.pay_off; o < end; ++cnt) {
        if (cnt == 17) return false;
        Item it;
        const uint32_t n = rlp_item(node + o, end - o, it);
        if (n == 0) return false;
        if (cnt == 0) { i0 = it; o0 = o; }
        if (cnt == 1) { i1 = it; o1 = o; }
        o += n;
    }
    if (cnt == 17) {
        uint32_t o = top.pay_off;
        for (uint32_t v = 0; v < 17; ++v) {
            Item it;
            const uint32_t n = rlp_item(node + o, end - o, it);
            if (v < 16) {
                if (!tn_child(it, o, t.c_kind[v], t.c_off[v], t.c_len[v])) return false;
            } else if (it.is_list || it.pay_len) return false;
            o += n;
        }
        t.kind = TN_BRANCH;
        return true;
    }
    if (cnt != 2 || i0.is_list || i0.pay_len == 0) return false;
    const uint8_t* hp = node + o0 + i0.pay_off;
    const uint32_t flag = hp[0] >> 4;
    if (flag > 3 || (!(flag & 1) && (hp[0] & 15))) return false;
    t.odd = flag & 1;
    t.path_off = o0 + i0.pay_off;
    t.plen = 2 * (i0.pay_len - 1) + t.odd;
    if (t.plen > 64) return false;
    if (flag & 2) {
        if (i1.is_list) return false;
        t.val_off = o1 + i1.pay_off;
        t.val_len = i1.pay_len;
        t.kind = TN_LEAF;
        return true;
    }
    if (t.plen == 0 || !tn_child(i1, o1, t.c_kind[0], t.c_off[0], t.c_len[0]) || t.c_kind[0] == TC_EMPTY) return false;
    t.kind = TN_EXT;
    return true;
}

// nibble q (< 64) of a 32-byte key
__device__ __forceinline__ uint32_t tk_nibble(const uint8_t* key, uint32_t q) { return (q & 1) ? (key[q >> 1] & 15u) : (key[q >> 1] >> 4); }
__device__ __forceinline__ void tk_set_nibble(uint8_t* key, uint32_t q, uint32_t v)
{
    uint8_t& b = key[q >> 1];
    b = (q & 1) ? (uint8_t)((b & 0xf0) | v) : (uint8_t)((b & 0x0f) | (v << 4));
}

// keys [lo, hi) (32 bytes each, sorted, all sharing their first `depth` nibbles): the sub-range whose nibbles
// [depth, depth + plen) equal the extension path of node `t`
__device__ void tk_ext_range(const uint8_t* keys, uint32_t lo, uint32_t hi, uint32_t depth, const uint8_t* node, const TNode& t,
                             uint32_t& sub_lo, uint32_t& sub_hi)
{
    for (int upper = 0; upper < 2; ++upper) {
        uint32_t a = lo, b = hi;
        while (a < b) {
            const uint32_t mid = (a + b) >> 1;
            int c = 0;
            for (uint32_t j = 0; j < t.plen && !c; ++j) {
                const uint32_t kn = tk_nibble(keys + 32ull * mid, depth + j), pn = tn_path_nibble(node, t, j);
                c = kn < pn ? -1 : (kn > pn ? 1 : 0);
            }
            if (upper ? c <= 0 : c < 0) a = mid + 1; else b = mid;
        }
        (upper ? sub_hi : sub_lo) = a;
    }
}

// keys [lo, hi) as above: the first key whose nibble `depth` is >= v
__device__ uint32_t tk_nibble_bound(const uint8_t* keys, uint32_t lo, uint32_t hi, uint32_t depth, uint32_t v)
{
    uint32_t a = lo, b = hi;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (tk_nibble(keys + 32ull * mid, depth) < v) a = mid + 1; else b = mid;
    }
    return a;
}

} // namespace
} // namespace phant
