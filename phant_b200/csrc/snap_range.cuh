// snap_range.cuh -- the per-request rules of the snap protocol's GetAccountRange and GetStorageRanges answers served from the
// resident world state (phant_gpu_resident_state_snap_ranges in include/phant_gpu.h), at the current root.  Device code,
// called by the snap-range kernels in trie.cu.  DESIGN.md §4.3m.
//
// The rules are go-ethereum's snap handler (ServiceGetAccountRangeQuery / ServiceGetStorageRangesQuery) over prefix sums:
//
//   sizes      an account entry is 32 + its slim body rlp([nonce, balance, root or "", codeHash or ""]); a slot entry is 32 +
//              rlp(trimmed value), the trie leaf's value.  So an account entry is at least 37 bytes and a slot entry 33.
//   windows    an account request's candidates are the row table's keys >= origin up to and including the first key >= limit
//              (at least one when any key >= origin exists), at most bytes / 37 + 1 of them: more entries than that cannot be
//              returned.  A storage request's candidates are, account after account, each account's slot keys >= o up to and
//              including the first >= l (o, l: the request's origin and limit for its first account, 0 and ff..ff after),
//              hard / 33 + 1 in all (hard = bytes + bytes / 10).
//   cuts       with x the exclusive prefix sum of the candidates' sizes: an account request keeps its candidates up to and
//              including the first whose running size is > bytes.  A storage request serves accounts while the running size is
//              < bytes; within an account it appends keys while the running size is < hard, and an account that stops on the
//              hard limit with keys left is cut.  The first account that carries a proof (o != 0, or cut with entries) ends
//              the reply.
//
// Templated on the row types (KRow and SlotRow in trie.cu), as resident_range.cuh, so that the whole statement compiles as
// HOST code (tests/hostcheck/snap_range_host.cpp).  Include phant_gpu.h first.
#pragma once
#include <stdint.h>

#include "resident_range.cuh" // rd_cmp32, rg_bound_rows, rg_bound_slots
#include "state_read.cuh"     // AccountBody, decode_account_body

namespace phant {
namespace {

// whether 32 bytes are the big-endian words w (immediates, so that this header adds nothing to the module's constant bank)
__device__ __forceinline__ bool snp_is(const uint8_t* p, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t w4, uint32_t w5,
                                       uint32_t w6, uint32_t w7)
{
    const uint32_t w[8] = {w0, w1, w2, w3, w4, w5, w6, w7};
    bool eq = true;
#pragma unroll
    for (int i = 0; i < 8; ++i) eq &= ((uint32_t)p[4 * i] << 24 | (uint32_t)p[4 * i + 1] << 16 | (uint32_t)p[4 * i + 2] << 8 | p[4 * i + 3]) == w[i];
    return eq;
}
// keccak(0x80), the empty trie's root, and keccak(""), the empty code's hash
__device__ __forceinline__ bool snp_empty_root(const uint8_t* p)
{
    return snp_is(p, 0x56e81f17u, 0x1bcc55a6u, 0xff8345e6u, 0x92c0f86eu, 0x5b48e01bu, 0x996cadc0u, 0x01622fb5u, 0xe363b421u);
}
__device__ __forceinline__ bool snp_empty_code(const uint8_t* p)
{
    return snp_is(p, 0xc5d24601u, 0x86f7233cu, 0x927e7db2u, 0xdcc703c0u, 0xe500b653u, 0xca82273bu, 0x7bfad804u, 0x5d85a470u);
}

constexpr uint32_t SNP_NONE = 0xffffffffu;

// the RLP string of n big-endian bytes without leading zeros (n == 0: the empty string)
__device__ __forceinline__ uint32_t snp_str_len(const uint8_t* b, uint32_t n)
{
    return n == 1 && b[0] < 0x80 ? 1 : 1 + n;
}
__device__ __forceinline__ uint8_t* snp_put_str(uint8_t* o, const uint8_t* b, uint32_t n)
{
    if (!(n == 1 && b[0] < 0x80)) *o++ = (uint8_t)(0x80 + n);
    for (uint32_t i = 0; i < n; ++i) *o++ = b[i];
    return o;
}

// The slim body of the account leaf value `leaf` (len bytes): written to out when it is not null.  Returns its length, 0 when
// the leaf does not decode (cannot happen for the trie's own leaves).  At most 2 + 9 + 33 + 33 + 33 = 110 bytes.
__device__ __forceinline__ uint32_t snp_slim(const uint8_t* leaf, uint32_t len, uint8_t* out)
{
    AccountBody a;
    if (!decode_account_body(leaf, len, a)) return 0;
    uint32_t nn = 0; // the nonce's big-endian bytes without leading zeros
    while (nn < 8 && (a.nonce >> (8 * nn))) ++nn;
    const bool er = snp_empty_root(leaf + a.root_off), ec = snp_empty_code(leaf + a.code_off);
    const uint32_t pay = (nn == 1 && a.nonce < 0x80 ? 1 : 1 + nn) + snp_str_len(leaf + a.bal_off, a.bal_len) + (er ? 1 : 33) + (ec ? 1 : 33);
    const uint32_t hdr = pay <= 55 ? 1 : 2;
    if (out) {
        uint8_t* o = out;
        if (hdr == 1) *o++ = (uint8_t)(0xc0 + pay);
        else { *o++ = 0xf8; *o++ = (uint8_t)pay; }
        if (!(nn == 1 && a.nonce < 0x80)) *o++ = (uint8_t)(0x80 + nn);
        for (uint32_t i = nn; i-- > 0;) *o++ = (uint8_t)(a.nonce >> (8 * i));
        o = snp_put_str(o, leaf + a.bal_off, a.bal_len);
        o = snp_put_str(o, leaf + a.root_off, er ? 0 : 32);
        snp_put_str(o, leaf + a.code_off, ec ? 0 : 32);
    }
    return hdr + pay;
}

// A slot's body rlp(trimmed value) from its 32-byte value (never zero in the table), written to out when it is not null.
__device__ __forceinline__ uint32_t snp_slot_body(const uint8_t* v, uint8_t* out)
{
    uint32_t z = 0;
    while (z < 32 && v[z] == 0) ++z;
    if (out) snp_put_str(out, v + z, 32 - z);
    return snp_str_len(v + z, 32 - z);
}

// the storage budget's hard limit: bytes * 1.1 in integers, saturated
__device__ __forceinline__ uint64_t snp_hard(uint64_t bytes)
{
    const uint64_t h = bytes + bytes / 10;
    return h < bytes ? ~0ull : h;
}
// the most entries a budget can return: an account entry is at least 37 bytes, a slot entry at least 33
__device__ __forceinline__ uint64_t snp_account_cap(uint64_t bytes) { return bytes / 37 + 1; }
__device__ __forceinline__ uint64_t snp_slot_cap(uint64_t hard) { return hard / 33 + 1; }

// the run [lo, lo + cnt) of n sorted keys found at [lo, first_ge_limit]: from the first key >= origin up to and including the
// first key >= limit (one key when origin > limit), given the bounds the caller found
__device__ __forceinline__ uint64_t snp_run(uint32_t lo, uint32_t lim_lb, uint32_t end)
{
    if (lo >= end) return 0;
    const uint32_t ub = lim_lb < end ? lim_lb + 1 : end;
    return (ub > lo ? ub : lo + 1) - lo;
}

// An account request's candidates: rows [lo, lo + cnt) of the account trie's row table
template <class KRowT>
__device__ void snp_account_window(const KRowT* rows, uint32_t n, const uint8_t* origin, const uint8_t* limit, uint64_t bytes, uint32_t& lo,
                                   uint64_t& cnt)
{
    lo = rg_bound_rows(rows, n, origin, false);
    const uint64_t run = snp_run(lo, rg_bound_rows(rows, n, limit, false), n), cap = snp_account_cap(bytes);
    cnt = run < cap ? run : cap;
}

// Slot keys of account akey in the slot table (sorted by (account, slot)): the run from the first key >= o up to and including
// the first >= l, starting at row lo
template <class SlotRowT>
__device__ void snp_slot_run(const SlotRowT* S, uint32_t nS, const uint8_t* akey, const uint8_t* o, const uint8_t* l, uint32_t& lo, uint64_t& run)
{
    uint8_t ff[32];
    for (int b = 0; b < 32; ++b) ff[b] = 0xff;
    const uint32_t end = rg_bound_slots(S, nS, akey, ff, true);
    lo = rg_bound_slots(S, nS, akey, o, false);
    run = snp_run(lo, rg_bound_slots(S, nS, akey, l, false), end);
}

// A storage request's candidates over its na accounts (accts: na x 32): per account its first row, run and candidates; the
// candidates stop at the request's cap.  Once the cap is reached the later accounts are not searched: a walk that appended
// every candidate has a running size of at least 33 * cap > hard >= bytes, so snp_storage_cut never serves them.
template <class SlotRowT>
__device__ void snp_storage_window(const SlotRowT* S, uint32_t nS, const uint8_t* accts, uint64_t na, const uint8_t* origin, const uint8_t* limit,
                                   uint64_t bytes, uint32_t* lo, uint64_t* run, uint64_t* cand)
{
    uint8_t zero[32], ff[32];
    for (int b = 0; b < 32; ++b) { zero[b] = 0; ff[b] = 0xff; }
    uint64_t left = snp_slot_cap(snp_hard(bytes));
    for (uint64_t k = 0; k < na; ++k) {
        if (left == 0) { lo[k] = 0; run[k] = cand[k] = 0; continue; }
        snp_slot_run(S, nS, accts + 32ull * k, k ? zero : origin, k ? ff : limit, lo[k], run[k]);
        cand[k] = run[k] < left ? run[k] : left;
        left -= cand[k];
    }
}

// An account request's entries: x is the exclusive prefix of its cnt candidates' sizes (x[0] the base); the first j >= 1 with
// x[j] - x[0] > bytes, or cnt
__device__ __forceinline__ uint64_t snp_account_cut(const uint64_t* x, uint64_t cnt, uint64_t bytes)
{
    uint64_t a = 1, b = cnt; // the answer lies in [a, b] when cnt > 0
    if (cnt == 0) return 0;
    while (a < b) {
        const uint64_t mid = a + ((b - a) >> 1);
        if (x[mid] - x[0] > bytes) b = mid; else a = mid + 1;
    }
    return a;
}

// A storage request's answer: accounts served, the one carrying a proof (SNP_NONE: none) and whether it is cut
struct SnpServe {
    uint64_t served;
    uint32_t proved;
    bool cut;
};
// x: the exclusive prefix of the request's candidates' sizes, account after account (x[0] the base); cand / run per account
// (snp_storage_window); origin_set: the request's origin is not zero.  ent receives each account's entries (0 once it is not
// served).
__device__ inline SnpServe snp_storage_cut(const uint64_t* x, const uint64_t* cand, const uint64_t* run, uint64_t na, bool origin_set,
                                           uint64_t bytes, uint64_t* ent)
{
    const uint64_t hard = snp_hard(bytes);
    SnpServe r{0, SNP_NONE, false};
    uint64_t t0 = 0, size = 0;
    for (uint64_t k = 0; k < na; ++k) ent[k] = 0;
    for (uint64_t k = 0; k < na; ++k) {
        if (size >= bytes) break;
        r.served = k + 1;
        // the first candidate of this account whose running size before it is >= hard, or its end
        uint64_t a = t0, b = t0 + cand[k];
        while (a < b) {
            const uint64_t mid = a + ((b - a) >> 1);
            if (x[mid] - x[0] >= hard) b = mid; else a = mid + 1;
        }
        ent[k] = a - t0;
        size = x[a] - x[0];
        const bool cut = ent[k] < run[k];
        if ((k == 0 && origin_set) || (cut && ent[k] > 0)) {
            r.proved = (uint32_t)k;
            r.cut = cut;
            break;
        }
        t0 += cand[k];
    }
    return r;
}

} // namespace
} // namespace phant
