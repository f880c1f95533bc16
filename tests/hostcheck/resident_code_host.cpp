// Test-only: compiles the DEVICE per-item statements of the resident code store (phant_b200/csrc/resident_code.cuh, on top
// of resident_read.cuh) as HOST code -- CUDA qualifiers and intrinsics defined away below, as in resident_read_host.cpp --
// and runs them the way the code kernels in trie.cu do: one lookup per hash, and a prune's marks from the current account
// rows and from every entry of the window's undo records.  Built as a shared object by
// tests/test_resident_code_header_host.py; nothing in the product links or loads this.
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
#include "phant_gpu.h"
#include "resident_code.cuh"

using namespace phant;

// the row layout of trie.cu (the account trie's rows and the code table's)
struct alignas(16) KRow { uint8_t key[32]; uint64_t off; uint32_t len; uint8_t cache[33]; };
static_assert(sizeof(KRow) == 80, "row layout");
static_assert(sizeof(RdRec) == 80, "descriptor layout");

// the code `hash` names in the table (n rows sorted by key): status; its arena slice
extern "C" int hc_lookup(const KRow* rows, uint32_t n, const uint8_t* hash, uint64_t* off, uint32_t* len)
{
    const CdCode c = cd_lookup(rows, n, hash);
    *off = c.off;
    *len = c.len;
    return (int)c.status;
}

// a prune's marks: keep[i] = 1 when code row i is named by a current account row (nK rows, bodies in arena) or by an entry of
// the `back` records.  Returns 1 when an account body does not decode.
extern "C" int hc_marks(const KRow* krows, uint32_t nK, const uint8_t* arena, const RdRec* recs, uint32_t back, const KRow* rows, uint32_t n,
                        uint8_t* keep)
{
    int bad = 0;
    memset(keep, 0, n);
    for (uint32_t i = 0; i < nK; ++i) {
        const uint8_t* h = cd_account_code(krows, i, arena);
        if (!h) { bad = 1; continue; }
        cd_mark(rows, n, h, keep);
    }
    for (uint32_t k = 0; k < back; ++k)
        for (uint32_t p = 0; p < recs[k].na; ++p) cd_mark(rows, n, cd_record_code(recs[k], p), keep);
    return bad;
}
