// state_read.cu -- pre-state reads from an execution witness (entry point P of include/phant_gpu.h).
//
// Two passes over the node set that entry point W hashed and put into its digest table (abi.cu runs both steps first):
//   account pass: one account key per thread -- the W walk from the state root, the account body decoded
//                 (state_read.cuh), the code looked up by codeHash in a second table over keccak(codes[i]); it leaves a
//                 record per account (status + storage root) in device memory;
//   slot pass:    one slot key per thread -- gathers its account's record and walks from that storage root through the same
//                 node table, then decodes the value.
// The storage roots never leave the device, so a slot is only ever proven under the root its account leaf holds.
// Rules: DESIGN.md "P: pre-state reads"; test statement: tests/state_read_oracle.py.
#include "common.cuh"

#include "../../include/phant_gpu.h"
#include "state_read.cuh" // (includes walk_one.cuh: walk_one<BAG>, bag_find, load32 ...)

namespace phant {
namespace {

// keccak256("") -- the codeHash of an account without code
__constant__ uint8_t EMPTY_CODE_HASH[32] = {0xc5, 0xd2, 0x46, 0x01, 0x86, 0xf7, 0x23, 0x3c, 0x92, 0x7e, 0x7d, 0xb2, 0xdc, 0xc7, 0x03, 0xc0,
                                            0xe5, 0x00, 0xb6, 0x53, 0xca, 0x82, 0x27, 0x3b, 0x7b, 0xfa, 0xd8, 0x04, 0x5d, 0x85, 0xa4, 0x70};

// 32 bytes held as 8 little-endian words (load32's layout) -> dst; two 128-bit stores when dst allows it
__device__ __forceinline__ void store32(uint8_t* dst, const uint32_t (&w)[8])
{
    if (!((uintptr_t)dst & 15)) {
        reinterpret_cast<uint4*>(dst)[0] = make_uint4(w[0], w[1], w[2], w[3]);
        reinterpret_cast<uint4*>(dst)[1] = make_uint4(w[4], w[5], w[6], w[7]);
        return;
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) dst[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
}

// n (<= 32) big-endian bytes at src, left padded to 32 bytes, as 8 little-endian words (unrolled: no dynamic register index)
__device__ __forceinline__ void pad32(const uint8_t* src, uint32_t n, uint32_t (&w)[8])
{
    const int lead = 32 - (int)n;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint32_t v = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = 4 * i + j - lead;
            if (k >= 0) v |= (uint32_t)src[k] << (8 * j);
        }
        w[i] = v;
    }
}

__global__ void __launch_bounds__(128, 6)
read_accounts_kernel(const Bag bag, uint64_t n, const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off,
                     const uint8_t* __restrict__ digests, const uint32_t* __restrict__ summary, const uint8_t* __restrict__ keys32,
                     const uint8_t* __restrict__ roots32, uint64_t n_roots, const Bag code_bag, const uint8_t* __restrict__ code_digests,
                     uint8_t* __restrict__ rec_roots32, uint8_t* __restrict__ rec_status, const StateOut out)
{
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t vo;
        uint32_t vl;
        int st = walk_one<true>(nodes, node_off, nullptr, bag, 0, 0, keys32 + 32 * i, roots32 + (n_roots == 1 ? 0 : 32 * i), digests, summary,
                                vo, vl);
        AccountBody a{};
        if (st == ST_PRESENT && !decode_account_body(nodes + vo, vl, a)) st = ST_REJECT;
        uint32_t root[8] = {0, 0, 0, 0, 0, 0, 0, 0}, code[8] = {0, 0, 0, 0, 0, 0, 0, 0}, bal[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint32_t ci = PHANT_GPU_CODE_EMPTY;
        if (st == ST_PRESENT) {
            const uint8_t* body = nodes + vo;
            load32(body + a.root_off, root); // inside the node: the 16-byte slack rule of load32 holds
            load32(body + a.code_off, code);
            pad32(body + a.bal_off, a.bal_len, bal);
            if (!eq32_const(EMPTY_CODE_HASH, code)) {
                ci = PHANT_GPU_CODE_MISSING;
                if (code_bag.table) {
                    const uint32_t f = bag_find(code_bag, code_digests, code);
                    if (f != BAG_EMPTY) ci = f;
                }
            }
        } else {
            a.nonce = 0;
        }
        store32(rec_roots32 + 32 * i, root);
        rec_status[i] = (uint8_t)st;
        if (out.account_status) out.account_status[i] = (uint8_t)st;
        if (out.nonce) out.nonce[i] = a.nonce;
        if (out.balance32) store32(out.balance32 + 32 * i, bal);
        if (out.storage_root32) store32(out.storage_root32 + 32 * i, root);
        if (out.code_hash32) store32(out.code_hash32 + 32 * i, code);
        if (out.code_index) out.code_index[i] = ci;
    }
}

__global__ void __launch_bounds__(128, 6)
read_slots_kernel(const Bag bag, uint64_t n, const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off,
                  const uint8_t* __restrict__ digests, const uint32_t* __restrict__ summary, const uint8_t* __restrict__ keys32,
                  const uint32_t* __restrict__ slot_account, uint64_t n_accounts, const uint8_t* __restrict__ rec_roots32,
                  const uint8_t* __restrict__ rec_status, const StateOut out)
{
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t acc = slot_account[i];
        int st = ST_REJECT; // an account index out of range (device pointers are not validated)
        uint32_t val[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (acc < n_accounts) {
            st = rec_status[acc]; // absent account: all its storage is absent; 0 / 3: passed on, not walked
            if (st == ST_PRESENT) {
                uint64_t vo;
                uint32_t vl, off, len;
                // an empty storage root gives ST_ABSENT without a lookup (walk_one)
                st = walk_one<true>(nodes, node_off, nullptr, bag, 0, 0, keys32 + 32 * i, rec_roots32 + 32 * acc, digests, summary, vo, vl);
                if (st == ST_PRESENT) {
                    if (decode_slot_value(nodes + vo, vl, off, len)) pad32(nodes + vo + off, len, val);
                    else st = ST_REJECT;
                }
            }
        }
        if (out.slot_status) out.slot_status[i] = (uint8_t)st;
        if (out.slot_vals32) store32(out.slot_vals32 + 32 * i, val);
    }
}

unsigned walk_blocks(int device, uint64_t n)
{
    uint64_t blocks = (n + 127) / 128;
    const uint64_t cap = (uint64_t)keccak_num_sms(device) * 16;
    if (blocks > cap) blocks = cap;
    return blocks ? (unsigned)blocks : 1u; // one (idle) CTA for an empty list: the launch sequence does not depend on the counts
}

} // namespace

cudaError_t launch_read_accounts(cudaStream_t s, int device, uint64_t n_accounts, const uint8_t* nodes, const uint64_t* node_off,
                                 const uint8_t* digests, const uint32_t* summary, const uint32_t* table, uint32_t capacity,
                                 const uint8_t* keys32, const uint8_t* roots32, uint64_t n_roots, const uint8_t* code_digests,
                                 const uint32_t* code_table, uint32_t code_capacity, uint8_t* rec_roots32, uint8_t* rec_status,
                                 const StateOut& out)
{
    read_accounts_kernel<<<walk_blocks(device, n_accounts), 128, 0, s>>>(
        Bag{table, capacity - 1}, n_accounts, nodes, node_off, digests, summary, keys32, roots32, n_roots,
        Bag{code_table, code_table ? code_capacity - 1 : 0}, code_digests, rec_roots32, rec_status, out);
    return cudaGetLastError();
}

cudaError_t launch_read_slots(cudaStream_t s, int device, uint64_t n_slots, const uint8_t* nodes, const uint64_t* node_off,
                              const uint8_t* digests, const uint32_t* summary, const uint32_t* table, uint32_t capacity,
                              const uint8_t* keys32, const uint32_t* slot_account, uint64_t n_accounts, const uint8_t* rec_roots32,
                              const uint8_t* rec_status, const StateOut& out)
{
    read_slots_kernel<<<walk_blocks(device, n_slots), 128, 0, s>>>(Bag{table, capacity - 1}, n_slots, nodes, node_off, digests, summary,
                                                                   keys32, slot_account, n_accounts, rec_roots32, rec_status, out);
    return cudaGetLastError();
}

} // namespace phant
