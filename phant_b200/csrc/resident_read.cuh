// resident_read.cuh -- one key's value in the resident world state (phant_gpu_resident_state_read in include/phant_gpu.h),
// as it is now or as it was `back` applies ago.  Per thread, device code, called by the read kernels in trie.cu.
//
//   now     an account: its row in the account trie's sorted row table (key, arena slice holding rlp([nonce, balance,
//           storageRoot, codeHash])), decoded by P's account decoder; a slot: its row in the slot table, sorted by
//           (account key, slot key).  No hashing.
//   past    the undo records of the last `back` applies, oldest first.  A record is the inverse diff of its apply: the old
//           fields of every account the apply listed (sorted by key), the old storage root of each, and the old values of
//           its slots (sorted by record account, then slot key).  The first record that lists the account, or covers the
//           slot, holds its value before the window; nothing covers it -> the value now.
//
// The row types are template parameters (KRow and SlotRow in trie.cu), so that the same statements can be compiled as HOST
// code by the test harness (tests/hostcheck/resident_read_host.cpp) and compared with a Python model of the state at every
// root a journal reaches, on a machine without a GPU.  Include phant_gpu.h first (the account flags).  DESIGN.md §4.3g.
#pragma once
#include <stdint.h>

#include "state_read.cuh" // AccountBody, decode_account_body

namespace phant {
namespace {

enum { RD_BAD = 0, RD_PRESENT = 1, RD_ABSENT = 2 };

// One undo record as it lies on the device: the diff arrays revert replays, then the old storage roots (32 B per account;
// zero for a DELETE account).
struct RdRec {
    const uint8_t *akeys, *aflags;
    const uint64_t* nonce;
    const uint8_t *bal, *code, *sroot;
    const uint32_t* sacc;
    const uint8_t *skeys, *svals;
    uint32_t na, ms;
};

// An account's value: where its fields are (bal: bal_len big-endian bytes; sroot and code: 32 bytes each).  Absent or bad:
// no field.
struct RdAccount {
    uint32_t status;
    uint64_t nonce;
    const uint8_t *bal, *sroot, *code;
    uint32_t bal_len;
};
// A slot's value: 32 bytes big endian, present only when not zero.
struct RdSlot {
    uint32_t status;
    const uint8_t* val;
};

__device__ __forceinline__ int rd_cmp32(const uint8_t* a, const uint8_t* b)
{
    for (int i = 0; i < 32; ++i)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
// index of `key` among n sorted 32-byte keys, or n
__device__ __forceinline__ uint32_t rd_find32(const uint8_t* keys, uint32_t n, const uint8_t* key)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (rd_cmp32(keys + 32ull * mid, key) < 0) a = mid + 1; else b = mid;
    }
    return a < n && rd_cmp32(keys + 32ull * a, key) == 0 ? a : n;
}

// listed slots [lo, hi) of listed account i, slots sorted by account: of a diff being applied (the undo capture), or of an
// undo record
__device__ __forceinline__ void listed_slots(const uint32_t* sacc, uint32_t ms, uint32_t i, uint32_t& lo, uint32_t& hi)
{
    uint32_t a = 0, b = ms;
    while (a < b) { const uint32_t mid = (a + b) >> 1; if (sacc[mid] < i) a = mid + 1; else b = mid; }
    uint32_t c = a, d = ms;
    while (c < d) { const uint32_t mid = (c + d) >> 1; if (sacc[mid] < i + 1) c = mid + 1; else d = mid; }
    lo = a;
    hi = c;
}

// The account as it is now: its row in the account trie's row table (n rows sorted by key, values in `arena`).
template <class KRowT> __device__ RdAccount rd_account_now(const KRowT* rows, uint32_t n, const uint8_t* arena, const uint8_t* key)
{
    RdAccount r{RD_ABSENT, 0, nullptr, nullptr, nullptr, 0};
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (rd_cmp32(rows[mid].key, key) < 0) a = mid + 1; else b = mid;
    }
    if (a == n || rd_cmp32(rows[a].key, key) != 0) return r;
    const uint8_t* body = arena + rows[a].off;
    AccountBody ab;
    if (!decode_account_body(body, rows[a].len, ab)) { r.status = RD_BAD; return r; }
    r.status = RD_PRESENT;
    r.nonce = ab.nonce;
    r.bal = body + ab.bal_off;
    r.bal_len = ab.bal_len;
    r.sroot = body + ab.root_off;
    r.code = body + ab.code_off;
    return r;
}

// The slot (akey, skey) as it is now: its row in the slot table (n rows sorted by (account key, slot key)).
template <class SlotRowT> __device__ RdSlot rd_slot_now(const SlotRowT* rows, uint32_t n, const uint8_t* akey, const uint8_t* skey)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        int c = rd_cmp32(rows[mid].akey, akey);
        if (c == 0) c = rd_cmp32(rows[mid].skey, skey);
        if (c < 0) a = mid + 1; else b = mid;
    }
    if (a < n && rd_cmp32(rows[a].akey, akey) == 0 && rd_cmp32(rows[a].skey, skey) == 0) return RdSlot{RD_PRESENT, rows[a].val};
    return RdSlot{RD_ABSENT, nullptr};
}

// The account as it was before the `back` applies whose records are recs[0 .. back), oldest first.
template <class KRowT>
__device__ RdAccount rd_account(const RdRec* recs, uint32_t back, const KRowT* rows, uint32_t n, const uint8_t* arena, const uint8_t* key)
{
    for (uint32_t k = 0; k < back; ++k) {
        const RdRec& R = recs[k];
        const uint32_t p = rd_find32(R.akeys, R.na, key);
        if (p == R.na) continue;
        if (R.aflags[p] & PHANT_GPU_ACCOUNT_DELETE) return RdAccount{RD_ABSENT, 0, nullptr, nullptr, nullptr, 0};
        return RdAccount{RD_PRESENT, R.nonce[p], R.bal + 32ull * p, R.sroot + 32ull * p, R.code + 32ull * p, 32};
    }
    return rd_account_now(rows, n, arena, key);
}

// The slot (akey, skey) as it was before the `back` applies whose records are recs[0 .. back), oldest first.  A record
// covers the slot when it lists the account with DELETE (absent) or CLEAR_STORAGE (it lists every slot the account had), or
// lists the slot itself (zero: absent).
template <class SlotRowT>
__device__ RdSlot rd_slot(const RdRec* recs, uint32_t back, const SlotRowT* rows, uint32_t n, const uint8_t* akey, const uint8_t* skey)
{
    for (uint32_t k = 0; k < back; ++k) {
        const RdRec& R = recs[k];
        const uint32_t p = rd_find32(R.akeys, R.na, akey);
        if (p == R.na) continue;
        const uint8_t f = R.aflags[p];
        if (f & PHANT_GPU_ACCOUNT_DELETE) return RdSlot{RD_ABSENT, nullptr};
        uint32_t lo, hi;
        listed_slots(R.sacc, R.ms, p, lo, hi);
        const uint32_t q = rd_find32(R.skeys + 32ull * lo, hi - lo, skey);
        if (q < hi - lo) {
            const uint8_t* v = R.svals + 32ull * (lo + q);
            uint32_t nz = 0;
            for (int b = 0; b < 32; ++b) nz |= v[b];
            return nz ? RdSlot{RD_PRESENT, v} : RdSlot{RD_ABSENT, nullptr};
        }
        if (f & PHANT_GPU_ACCOUNT_CLEAR_STORAGE) return RdSlot{RD_ABSENT, nullptr};
    }
    return rd_slot_now(rows, n, akey, skey);
}

} // namespace
} // namespace phant
