// Test-only: compiles the DEVICE decoders of pre-state reads (phant_b200/csrc/state_read.cuh) as HOST code -- CUDA
// qualifiers and the intrinsics walk_one.cuh uses are defined away below, as in walk_host.cpp -- so that the exact statements
// the GPU runs per account and per slot can be compared with the test decoders on a machine without a GPU.  Built as a shared
// object by tests/test_state_read_header_host.py; nothing in the product links or loads this.
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
#include "../../phant_b200/csrc/state_read.cuh"

using namespace phant;

// 1 + (nonce, balance offset / length, root offset, code offset) when the body follows the rules, 0 otherwise
extern "C" int hs_decode_account(const uint8_t* p, uint32_t len, uint64_t* nonce, uint32_t* f)
{
    AccountBody a{};
    if (!decode_account_body(p, len, a)) return 0;
    *nonce = a.nonce;
    f[0] = a.bal_off; f[1] = a.bal_len; f[2] = a.root_off; f[3] = a.code_off;
    return 1;
}

// 1 + (value offset, length) when the slot value follows the rules, 0 otherwise
extern "C" int hs_decode_slot(const uint8_t* p, uint32_t len, uint32_t* f)
{
    return decode_slot_value(p, len, f[0], f[1]) ? 1 : 0;
}
