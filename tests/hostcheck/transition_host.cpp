// Test-only: compiles the DEVICE node decoder of the transition roots (phant_b200/csrc/transition.cuh) as HOST code -- CUDA
// qualifiers and the intrinsics walk_one.cuh uses are defined away below, as in walk_host.cpp -- so that the exact statement the
// GPU runs per node can be compared with tests/transition_oracle.py on a machine without a GPU.  Built as a shared object by
// tests/test_transition_header_host.py; nothing in the product links or loads this.
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
#include "../../phant_b200/csrc/transition.cuh"

using namespace phant;

// kind (0 = breaks the rules); path nibbles into path[64] (count in *plen); f = value offset / length, then per child
// (kind, offset, length) x 16
extern "C" int ht_decode(const uint8_t* node, uint32_t len, uint8_t* path, uint32_t* plen, uint32_t* f)
{
    TNode t{};
    if (!tn_decode(node, len, t)) return 0;
    *plen = 0;
    if (t.kind != TN_BRANCH) {
        *plen = t.plen;
        for (uint32_t j = 0; j < t.plen; ++j) path[j] = (uint8_t)tn_path_nibble(node, t, j);
    }
    f[0] = t.val_off; f[1] = t.val_len;
    const uint32_t nc = t.kind == TN_BRANCH ? 16 : t.kind == TN_EXT ? 1 : 0;
    for (uint32_t v = 0; v < nc; ++v) { f[2 + 3 * v] = t.c_kind[v]; f[3 + 3 * v] = t.c_off[v]; f[4 + 3 * v] = t.c_len[v]; }
    return (int)t.kind;
}
