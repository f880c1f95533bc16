// resident_code.cuh -- contract code kept beside the resident world state (phant_gpu_resident_state_put_codes / _codes /
// _prune_codes in include/phant_gpu.h): what one hash looks up, and which accounts keep a code when the store is pruned.  Per
// item, device code, called by the code kernels in trie.cu.
//
//   store   a row table sorted by codeHash (KRow in trie.cu: key = keccak(code), off and len into a code arena).  The empty
//           code is never stored: keccak("") always counts as held, with length 0.
//   prune   a held code stays when an account names it at a root the journal reaches: a current account row (its body
//           decoded by P's decoder), or an entry of one of the window's undo records that is not DELETE -- the old codeHash of
//           an account present before that apply.  A DELETE entry is an account that was absent before its apply; its code
//           field means nothing and marks nothing.
//
// The row types are template parameters, as in resident_read.cuh, so that the same statements compile as HOST code in the
// test harness (tests/hostcheck/resident_code_host.cpp) and are compared there with a model of the store across block
// sequences.  Include phant_gpu.h first (the account flags).  DESIGN.md §4.3i.
#pragma once
#include <stdint.h>

#include "resident_read.cuh" // RdRec, rd_cmp32, AccountBody, decode_account_body

namespace phant {
namespace {

enum { CD_HELD = 1, CD_NOT_HELD = 2 };

__constant__ uint8_t CD_EMPTY_CODE_HASH[32] = {0xc5, 0xd2, 0x46, 0x01, 0x86, 0xf7, 0x23, 0x3c, 0x92, 0x7e, 0x7d, 0xb2, 0xdc, 0xc7, 0x03, 0xc0,
                                               0xe5, 0x00, 0xb6, 0x53, 0xca, 0x82, 0x27, 0x3b, 0x7b, 0xfa, 0xd8, 0x04, 0x5d, 0x85, 0xa4, 0x70};

// A hash's code: status, and its slice of the arena (length 0 for keccak("") and for a code that is not held).
struct CdCode {
    uint32_t status;
    uint32_t len;
    uint64_t off;
};

// index of the row keyed `hash` among n rows sorted by key, or n
template <class Row> __device__ uint32_t cd_find(const Row* rows, uint32_t n, const uint8_t* hash)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (rd_cmp32(rows[mid].key, hash) < 0) a = mid + 1; else b = mid;
    }
    return a < n && rd_cmp32(rows[a].key, hash) == 0 ? a : n;
}

template <class Row> __device__ CdCode cd_lookup(const Row* rows, uint32_t n, const uint8_t* hash)
{
    const uint32_t a = cd_find(rows, n, hash);
    if (a < n) return CdCode{CD_HELD, rows[a].len, rows[a].off};
    return CdCode{rd_cmp32(hash, CD_EMPTY_CODE_HASH) == 0 ? (uint32_t)CD_HELD : (uint32_t)CD_NOT_HELD, 0, 0};
}

// the codeHash current account row i names (the account trie's rows: values are account bodies in `arena`); nullptr when
// the body does not decode
template <class KRowT> __device__ const uint8_t* cd_account_code(const KRowT* rows, uint32_t i, const uint8_t* arena)
{
    const uint8_t* body = arena + rows[i].off;
    AccountBody b;
    return decode_account_body(body, rows[i].len, b) ? body + b.code_off : nullptr;
}

// the codeHash entry p of undo record R names, or nullptr for a DELETE entry
__device__ __forceinline__ const uint8_t* cd_record_code(const RdRec& R, uint32_t p)
{
    return (R.aflags[p] & PHANT_GPU_ACCOUNT_DELETE) ? nullptr : R.code + 32ull * p;
}

// keep the held code `hash` names (nullptr: none)
template <class Row> __device__ void cd_mark(const Row* rows, uint32_t n, const uint8_t* hash, uint8_t* keep)
{
    if (!hash) return;
    const uint32_t a = cd_find(rows, n, hash);
    if (a < n) keep[a] = 1;
}

} // namespace
} // namespace phant
