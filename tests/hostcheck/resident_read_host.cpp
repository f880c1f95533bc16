// Test-only: compiles the DEVICE per-key reads of the resident world state (phant_b200/csrc/resident_read.cuh) as HOST code --
// CUDA qualifiers and the intrinsics walk_one.cuh uses are defined away below, as in state_read_host.cpp -- so that the exact
// statements the GPU runs per account and per slot, now and through the undo records, can be compared with a model of the
// state at every root a journal reaches on a machine without a GPU.  Built as a shared object by
// tests/test_resident_read_header_host.py; nothing in the product links or loads this.
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
#include "../../include/phant_gpu.h"
#include "../../phant_b200/csrc/resident_read.cuh"

using namespace phant;

// the row layouts of trie.cu
struct alignas(16) KRow { uint8_t key[32]; uint64_t off; uint32_t len; uint8_t cache[33]; };
struct alignas(16) SlotRow { uint8_t akey[32], skey[32], val[32]; };
static_assert(sizeof(KRow) == 80 && sizeof(SlotRow) == 96, "row layout");
static_assert(sizeof(RdRec) == 80, "descriptor layout");

// the account `key` as it was `back` records ago (recs oldest first): status; nonce; balance, storage root, code hash (32 B
// each, big endian)
extern "C" int hr_account(const KRow* rows, uint32_t n, const uint8_t* arena, const RdRec* recs, uint32_t back, const uint8_t* key,
                          uint64_t* nonce, uint8_t* out96)
{
    const RdAccount a = rd_account(recs, back, rows, n, arena, key);
    const bool ok = a.status == RD_PRESENT;
    *nonce = ok ? a.nonce : 0;
    for (uint32_t b = 0; b < 32; ++b) {
        out96[b] = ok && b >= 32 - a.bal_len ? a.bal[b - (32 - a.bal_len)] : 0;
        out96[32 + b] = ok ? a.sroot[b] : 0;
        out96[64 + b] = ok ? a.code[b] : 0;
    }
    return (int)a.status;
}

// the slot (akey, skey) as it was `back` records ago: status; value (32 B)
extern "C" int hr_slot(const SlotRow* rows, uint32_t n, const RdRec* recs, uint32_t back, const uint8_t* akey, const uint8_t* skey, uint8_t* out32)
{
    const RdSlot v = rd_slot(recs, back, rows, n, akey, skey);
    for (uint32_t b = 0; b < 32; ++b) out32[b] = v.status == RD_PRESENT ? v.val[b] : 0;
    return (int)v.status;
}
