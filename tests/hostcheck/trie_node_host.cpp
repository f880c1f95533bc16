// Test-only: compiles the DEVICE walk by nibble path of the resident state's trie nodes (phant_b200/csrc/proof_chain.cuh,
// pc_node_at) as HOST code -- CUDA qualifiers and the intrinsics walk_one.cuh uses are defined away below, as in
// proof_chain_host.cpp -- so that the exact statement the GPU runs per path can be compared with the CPU statement
// (tests/trie_node_model.py) on a machine without a GPU.  Built as a shared object by tests/test_trie_node_header_host.py;
// nothing in the product links or loads this.
#include <stdint.h>
#include <string.h>
#define __device__
#define __forceinline__ inline
#define __constant__ static const
#define __restrict__
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 __ldg(const uint4* p) { uint4 v; memcpy(&v, p, sizeof v); return v; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t n) { n &= 31; return n ? (lo >> n) | (hi << (32 - n)) : lo; }
#include "../../phant_b200/csrc/proof_chain.cuh"

using namespace phant;

// n paths (32 bytes each, plen nibbles) under `root` over the set of m nodes sorted by digest: status and node index per path
extern "C" void hp_node_at(const uint8_t* bytes, const uint64_t* off, const uint8_t* dig, uint32_t m, const uint8_t* root,
                           const uint8_t* empty_root, const uint8_t* paths, const uint8_t* plen, uint32_t n, uint8_t* status,
                           uint32_t* index)
{
    const PcSet s{bytes, off, dig, m};
    for (uint32_t p = 0; p < n; ++p) {
        const PcAt a = pc_node_at(s, root, empty_root, paths + 32ull * p, plen[p]);
        status[p] = (uint8_t)a.status;
        index[p] = a.index;
    }
}
