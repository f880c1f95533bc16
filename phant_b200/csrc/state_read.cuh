// state_read.cuh -- the decoders of entry point P (include/phant_gpu.h): what a proven account leaf value and a proven
// storage leaf value say.  Per thread, device code, called by the kernels in state_read.cu.
//
// Kept in a header of its own, like walk_one.cuh, so that the same statements can be compiled as HOST code by the test
// harness (tests/hostcheck/state_read_host.cpp) and compared with an independently written decoder on a machine without a
// GPU.  Rules: DESIGN.md "P: pre-state reads".
#pragma once
#include <stdint.h>

#include "walk_one.cuh" // Item / rlp_item: the canonical-RLP rules of the walk

namespace phant {
namespace {

// The account body rlp([nonce, balance, storageRoot, codeHash]) (evmone/test/state/mpt_hash.cpp:15-36).  Offsets are
// from the first byte of the body.
struct AccountBody {
    uint64_t nonce;
    uint32_t bal_off, bal_len; // 0..32 big-endian bytes, no leading zero
    uint32_t root_off;         // 32 bytes
    uint32_t code_off;         // 32 bytes
};

// `p` / `len` = the payload of the account leaf's value item.  It must be exactly one RLP list of exactly four canonical
// strings: nonce 0..8 bytes and balance 0..32 bytes without a leading zero byte, storageRoot and codeHash 32 bytes each.
__device__ __forceinline__ bool decode_account_body(const uint8_t* p, uint32_t len, AccountBody& a)
{
    Item top;
    const uint32_t tot = rlp_item(p, len, top);
    if (tot == 0 || tot != len || !top.is_list) return false;
    const uint32_t end = top.pay_off + top.pay_len;
    uint32_t o = top.pay_off, off[4], n[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (o >= end) return false; // fewer than four items
        Item it;
        const uint32_t t = rlp_item(p + o, end - o, it);
        if (t == 0 || it.is_list) return false;
        off[i] = o + it.pay_off;
        n[i] = it.pay_len;
        o += t;
    }
    if (o != end) return false; // a fifth item
    if (n[0] > 8 || (n[0] && p[off[0]] == 0)) return false;
    if (n[1] > 32 || (n[1] && p[off[1]] == 0)) return false;
    if (n[2] != 32 || n[3] != 32) return false;
    uint64_t nonce = 0;
    for (uint32_t i = 0; i < n[0]; ++i) nonce = (nonce << 8) | p[off[0] + i];
    a.nonce = nonce;
    a.bal_off = off[1];
    a.bal_len = n[1];
    a.root_off = off[2];
    a.code_off = off[3];
    return true;
}

// `p` / `len` = the payload of the storage leaf's value item: one canonical RLP string of 1..32 bytes whose first byte is
// not zero (rlp(trim(value)); zero values are never stored, src/state/statedb.zig:112-119).  -> the value bytes.
__device__ __forceinline__ bool decode_slot_value(const uint8_t* p, uint32_t len, uint32_t& off, uint32_t& n)
{
    Item it;
    const uint32_t tot = rlp_item(p, len, it);
    if (tot == 0 || tot != len || it.is_list || it.pay_len == 0 || it.pay_len > 32 || p[it.pay_off] == 0) return false;
    off = it.pay_off;
    n = it.pay_len;
    return true;
}

} // namespace
} // namespace phant
