// range_proof.cuh -- the per-range rules of the range-proof check (phant_gpu_verify_ranges, include/phant_gpu.h): which entries
// a range may hold, which items of the boundary proofs lie inside [origin, last] and are replaced by the entries, and when a
// kept item means that the trie holds a key above the range.  Per thread, device code, called by the range kernels in trie.cu.
//
// Kept in a header of its own, like transition.cuh, so that the same statements can be compiled as HOST code by the test
// harness (tests/hostcheck/range_proof_host.cpp) and compared with the CPU statement tests/range_proof_oracle.py on a machine
// without a GPU.  Rules: DESIGN.md §4.3j.
#pragma once
#include <stdint.h>

namespace phant {
namespace {

__device__ __forceinline__ int rp_cmp(const uint8_t* a, const uint8_t* b)
{
    for (int i = 0; i < 32; ++i) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}

// An entry of a range: a non-empty value, a key strictly above the previous entry's (prev == nullptr for the range's first
// entry) and, unless the range is WHOLE, at or above the origin.
__device__ __forceinline__ bool rp_entry_ok(const uint8_t* key, const uint8_t* prev, const uint8_t* origin, bool whole, uint64_t vlen)
{
    if (vlen == 0) return false;
    if (prev && rp_cmp(prev, key) >= 0) return false;
    return whole || rp_cmp(key, origin) >= 0;
}

// The range's upper edge key: its last entry's key, or ff..ff when it has no entry (an empty answer claims that no key at or
// after the origin exists).
__device__ __forceinline__ void rp_last(const uint8_t* last_entry, uint8_t* out)
{
    for (int b = 0; b < 32; ++b) out[b] = last_entry ? last_entry[b] : 0xff;
}

// Whether the keys under prefix `key` (its first `depth` nibbles, zero after; depth 64: one leaf key) all lie in
// [origin, last]: origin <= P00..0 and Pff..f <= last.  A proof item for which this holds is replaced by the entries.
__device__ __forceinline__ bool rp_inside(const uint8_t* key, uint32_t depth, const uint8_t* origin, const uint8_t* last)
{
    if (rp_cmp(key, origin) < 0) return false;
    for (uint32_t i = 0; i < 32; ++i) {
        const uint8_t b = 2 * i >= depth ? 0xff : 2 * i + 1 == depth ? (uint8_t)(key[i] | 0x0f) : key[i];
        if (b != last[i]) return b < last[i];
    }
    return true;
}

// A proof item kept (outside [origin, last]) lies wholly below the origin or wholly above `last`: a subtree with an edge key
// under it is expanded, never kept as a stub.  Above means that the trie holds a key after the range.
__device__ __forceinline__ bool rp_above(const uint8_t* key, const uint8_t* last) { return rp_cmp(key, last) > 0; }

} // namespace
} // namespace phant
