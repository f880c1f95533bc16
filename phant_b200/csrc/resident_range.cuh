// resident_range.cuh -- account and storage ranges of the resident world state (phant_gpu_resident_state_range in
// include/phant_gpu.h), as it is now or as it was `back` applies ago.  Device code, called by the range kernels in trie.cu.
//
// A range is [origin, limit] over 32-byte big-endian keys, at most `max` entries: the accounts, or the slots of one account.
//
//   parts      each range has back + 1 candidate parts: part 0 is a run of the current table (the account trie's row table,
//              or the slot table sorted by (account key, slot key)), part 1 + k the keys record k lists inside the range.
//   the rule   R = the record keys inside the range, summed over the window's records.  Part 0 holds the first
//              min(ub - lb, max + 1 + R) keys of the current table in range; the record parts hold all R record keys.  A key
//              present now but absent at the past root is listed by some record, so at most R current candidates drop out and
//              the first max + 1 keys present at the past root are all candidates.  A storage range whose account some record
//              lists with DELETE or CLEAR_STORAGE has no part 0: rd_slot never reaches the current table for that account.
//   resolve    the candidates sorted by (range, key), adjacent duplicates dropped, each resolved by rd_account / rd_slot
//              (resident_read.cuh); the present ones ranked within their range, ranks < max returned, more = present > max.
//   back = 0   no record: part 0 alone, already sorted, unique and present, so it is returned as it is (no sort, no resolve).
//
// Templated on the row types (KRow and SlotRow in trie.cu), as resident_read.cuh, so that the whole statement compiles as
// HOST code (tests/hostcheck/resident_range_host.cpp).  Include phant_gpu.h first.  DESIGN.md §4.3h.
#pragma once
#include <stdint.h>

#include "resident_read.cuh" // RdRec, rd_cmp32, listed_slots, rd_account, rd_slot

namespace phant {
namespace {

// first of n sorted 32-byte keys that is >= key (upper: > key)
__device__ __forceinline__ uint32_t rg_bound32(const uint8_t* keys, uint32_t n, const uint8_t* key, bool upper)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        const int c = rd_cmp32(keys + 32ull * mid, key);
        if (c < 0 || (upper && c == 0)) a = mid + 1; else b = mid;
    }
    return a;
}
// first account row whose key is >= key (upper: > key)
template <class KRowT> __device__ uint32_t rg_bound_rows(const KRowT* rows, uint32_t n, const uint8_t* key, bool upper)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        const int c = rd_cmp32(rows[mid].key, key);
        if (c < 0 || (upper && c == 0)) a = mid + 1; else b = mid;
    }
    return a;
}
// first slot row whose (account key, slot key) is >= (akey, skey) (upper: >)
template <class SlotRowT> __device__ uint32_t rg_bound_slots(const SlotRowT* rows, uint32_t n, const uint8_t* akey, const uint8_t* skey, bool upper)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        int c = rd_cmp32(rows[mid].akey, akey);
        if (c == 0) c = rd_cmp32(rows[mid].skey, skey);
        if (c < 0 || (upper && c == 0)) a = mid + 1; else b = mid;
    }
    return a;
}

// The parts of account range [origin, limit] (at most `max` entries) at the root `back` records ago (recs oldest first):
// part p is [lo[p], lo[p] + cnt[p]) of the current row table (p = 0) or of record p - 1's account keys.
template <class KRowT>
__device__ void rg_account_parts(const RdRec* recs, uint32_t back, const KRowT* rows, uint32_t n, const uint8_t* origin, const uint8_t* limit,
                                 uint32_t max, uint32_t* lo, uint64_t* cnt)
{
    const bool empty = rd_cmp32(origin, limit) > 0;
    uint64_t R = 0;
    for (uint32_t k = 0; k < back; ++k) {
        const uint32_t a = rg_bound32(recs[k].akeys, recs[k].na, origin, false), b = rg_bound32(recs[k].akeys, recs[k].na, limit, true);
        lo[1 + k] = a;
        cnt[1 + k] = empty ? 0 : b - a;
        R += cnt[1 + k];
    }
    const uint32_t a = rg_bound_rows(rows, n, origin, false), b = rg_bound_rows(rows, n, limit, true);
    const uint64_t want = (uint64_t)max + 1 + R;
    lo[0] = a;
    cnt[0] = empty ? 0 : (b - a < want ? b - a : want);
}

// The parts of the storage range [origin, limit] of account `akey`: part 0 of the slot table, part 1 + k of record k's slot
// keys (the slots it lists for akey).
template <class SlotRowT>
__device__ void rg_slot_parts(const RdRec* recs, uint32_t back, const SlotRowT* rows, uint32_t n, const uint8_t* akey, const uint8_t* origin,
                              const uint8_t* limit, uint32_t max, uint32_t* lo, uint64_t* cnt)
{
    const bool empty = rd_cmp32(origin, limit) > 0;
    bool now = true; // the current slot table is a source
    uint64_t R = 0;
    for (uint32_t k = 0; k < back; ++k) {
        const RdRec& Rk = recs[k];
        lo[1 + k] = 0;
        cnt[1 + k] = 0;
        const uint32_t p = rd_find32(Rk.akeys, Rk.na, akey);
        if (p == Rk.na) continue;
        if (Rk.aflags[p] & (PHANT_GPU_ACCOUNT_DELETE | PHANT_GPU_ACCOUNT_CLEAR_STORAGE)) now = false;
        uint32_t l, h;
        listed_slots(Rk.sacc, Rk.ms, p, l, h);
        const uint32_t a = l + rg_bound32(Rk.skeys + 32ull * l, h - l, origin, false), b = l + rg_bound32(Rk.skeys + 32ull * l, h - l, limit, true);
        lo[1 + k] = a;
        cnt[1 + k] = empty ? 0 : b - a;
        R += cnt[1 + k];
    }
    const uint32_t a = rg_bound_slots(rows, n, akey, origin, false), b = rg_bound_slots(rows, n, akey, limit, true);
    const uint64_t want = (uint64_t)max + 1 + R;
    lo[0] = a;
    cnt[0] = empty || !now ? 0 : (b - a < want ? b - a : want);
}

// candidate i of part p (lo: the part's first index): its key
template <class KRowT> __device__ const uint8_t* rg_account_key(const RdRec* recs, const KRowT* rows, uint32_t p, uint32_t lo, uint64_t i)
{
    return p == 0 ? rows[lo + i].key : recs[p - 1].akeys + 32ull * (lo + i);
}
template <class SlotRowT> __device__ const uint8_t* rg_slot_key(const RdRec* recs, const SlotRowT* rows, uint32_t p, uint32_t lo, uint64_t i)
{
    return p == 0 ? rows[lo + i].skey : recs[p - 1].skeys + 32ull * (lo + i);
}

// the segment that holds item j, given n + 1 non-decreasing offsets: the largest r < n with off[r] <= j
__device__ __forceinline__ uint64_t rg_segment(const uint64_t* off, uint64_t n, uint64_t j)
{
    uint64_t a = 0, b = n;
    while (b - a > 1) {
        const uint64_t mid = (a + b) >> 1;
        if (off[mid] <= j) a = mid; else b = mid;
    }
    return a;
}

// the candidate that is present entry t of a range whose sorted candidates are [b, e): x is the exclusive scan of the
// present flags, so it is the first j in [b, e) with x[j + 1] > x[b] + t
__device__ __forceinline__ uint64_t rg_nth_present(const uint64_t* x, uint64_t b, uint64_t e, uint64_t t)
{
    const uint64_t want = x[b] + t;
    while (b < e) {
        const uint64_t mid = (b + e) >> 1;
        if (x[mid + 1] <= want) b = mid + 1; else e = mid;
    }
    return b;
}

// a range with `present` keys at its root: the entries returned and whether more follow
__device__ __forceinline__ void rg_select(uint64_t present, uint32_t max, uint64_t& entries, uint8_t& more)
{
    entries = present < max ? present : max;
    more = present > max;
}

} // namespace
} // namespace phant
