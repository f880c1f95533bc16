// Test-only: compiles the DEVICE sources of the proof walk (phant_b200/csrc/walk_one.cuh) and of the node summary
// (node_summary.cuh) as HOST code -- CUDA qualifiers and the three intrinsics they use are defined away below -- so that the
// exact statements the GPU executes per thread can be fuzzed against the oracle on a machine without a GPU.  Built as a
// shared object by tests/test_walk_header_host.py; nothing in the product links or loads this.
#include <stdint.h>
#include <string.h>
#include <vector>
#define __device__
#define __forceinline__ inline
#define __constant__ static const
#define __restrict__
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 __ldg(const uint4* p) { uint4 v; memcpy(&v, p, sizeof v); return v; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t n) { n &= 31; return n ? (lo >> n) | (hi << (32 - n)) : lo; }
#include "../../phant_b200/csrc/node_summary.cuh"
#include "../../phant_b200/csrc/walk_one.cuh"

using namespace phant;

// summaries as the hash kernels would leave them: on == 1, the staged kernel (only nodes that fit its first window);
// on == 2, the direct kernel (every node up to 4096 bytes, read from global memory)
static std::vector<uint32_t> summaries(const uint8_t* nodes, const uint64_t* node_off, uint64_t n_nodes, int on)
{
    std::vector<uint32_t> s(n_nodes + 1, 0);
    if (on)
        for (uint64_t j = 0; j < n_nodes; ++j) {
            const uint64_t len = node_off[j + 1] - node_off[j];
            if (len <= (on == 2 ? 4096u : 544u)) s[j] = summarize_node(nodes + node_off[j], (uint32_t)len);
        }
    return s;
}

extern "C" int hostwalk_chain(const uint8_t* nodes, const uint64_t* node_off, uint64_t n_nodes, const uint64_t* node_index,
                              const uint64_t* proof_first, uint64_t n_proofs, const uint8_t* keys32, const uint8_t* roots32,
                              uint64_t n_roots, const uint8_t* digests, int use_summary, uint8_t* status, uint64_t* voff, uint32_t* vlen)
{
    const std::vector<uint32_t> sm = summaries(nodes, node_off, n_nodes, use_summary);
    for (uint64_t p = 0; p < n_proofs; ++p)
        status[p] = (uint8_t)walk_one<false>(nodes, node_off, node_index, Bag{nullptr, 0}, proof_first[p], proof_first[p + 1], keys32 + 32 * p,
                                             roots32 + (n_roots == 1 ? 0 : 32 * p), digests, use_summary ? sm.data() : nullptr, voff[p], vlen[p]);
    return 0;
}

extern "C" int hostwalk_bag(const uint8_t* nodes, const uint64_t* node_off, uint64_t n_nodes, uint64_t n_keys, const uint8_t* keys32,
                            const uint8_t* roots32, uint64_t n_roots, const uint8_t* digests, int use_summary, uint8_t* status,
                            uint64_t* voff, uint32_t* vlen)
{
    const std::vector<uint32_t> sm = summaries(nodes, node_off, n_nodes, use_summary);
    uint32_t capacity = 64;
    while (capacity < 2 * n_nodes) capacity <<= 1;
    std::vector<uint32_t> table(capacity, BAG_EMPTY);
    for (uint64_t i = 0; i < n_nodes; ++i) { // what bag_insert_kernel does, one thread at a time
        uint32_t e[8];
        load32_aligned(digests + 32 * i, e);
        uint32_t s = bag_slot(e, capacity - 1);
        for (;;) {
            if (table[s] == BAG_EMPTY) { table[s] = (uint32_t)i; break; }
            if (eq32_aligned(digests + 32ull * table[s], e)) break;
            s = (s + 1) & (capacity - 1);
        }
    }
    for (uint64_t p = 0; p < n_keys; ++p)
        status[p] = (uint8_t)walk_one<true>(nodes, node_off, nullptr, Bag{table.data(), capacity - 1}, 0, 0, keys32 + 32 * p,
                                            roots32 + (n_roots == 1 ? 0 : 32 * p), digests, use_summary ? sm.data() : nullptr, voff[p], vlen[p]);
    return 0;
}
