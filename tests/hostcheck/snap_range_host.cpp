// Test-only: compiles the DEVICE rules of the snap range answers (phant_b200/csrc/snap_range.cuh, on top of
// resident_range.cuh) as HOST code -- CUDA qualifiers defined away below, as in resident_range_host.cpp -- and runs one whole
// call's entries the way rs_snap_ranges in trie.cu runs them: every request's window, the candidates' sizes, one exclusive scan,
// every request's cut, and the fill of keys and bodies.  Built as a shared object by tests/test_snap_range_header_host.py;
// nothing in the product links or loads this.
#include <stdint.h>
#include <string.h>

#include <vector>
#define __device__
#define __forceinline__ inline
#define __constant__ static const
#define __restrict__
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 __ldg(const uint4* p) { uint4 v; memcpy(&v, p, sizeof v); return v; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t n) { n &= 31; return n ? (lo >> n) | (hi << (32 - n)) : lo; }
#include "phant_gpu.h"
#include "snap_range.cuh"

using namespace phant;

// the row layouts of trie.cu
struct alignas(16) KRow { uint8_t key[32]; uint64_t off; uint32_t len; uint8_t cache[33]; };
struct alignas(16) SlotRow { uint8_t akey[32], skey[32], val[32]; };
static_assert(sizeof(KRow) == 80 && sizeof(SlotRow) == 96, "row layout");

// One call: n account requests (origin, limit: n x 32; bytes: n), m storage requests over accounts [first[q], first[q + 1]) of
// accts (origin, limit: m x 32; bytes: m).  Out: ent (n + M: entries per account request, then per storage account), served
// and proved (m; proved = SNP_NONE when no account carries a proof), keys (32 B per entry, account entries first) and bodies
// (CSR: boff, one offset per entry + 1).  Returns 0, 1 when an account leaf does not decode, 2 when the output exceeds cap /
// bcap.
extern "C" int hs_snap(const KRow* krows, uint32_t nK, const uint8_t* arena, const SlotRow* S, uint32_t nS, uint32_t n, const uint8_t* aorigin,
                       const uint8_t* alimit, const uint64_t* abytes, uint32_t m, const uint64_t* first, const uint8_t* accts,
                       const uint8_t* sorigin, const uint8_t* slimit, const uint64_t* sbytes, uint64_t cap, uint64_t bcap, uint64_t* ent,
                       uint64_t* served, uint32_t* proved, uint8_t* keys, uint64_t* boff, uint8_t* bodies)
{
    const uint64_t M = m ? first[m] : 0, nseg = n + M;
    std::vector<uint32_t> lo(nseg);
    std::vector<uint64_t> cnt(nseg), run(M);
    for (uint32_t r = 0; r < n; ++r) snp_account_window(krows, nK, aorigin + 32ull * r, alimit + 32ull * r, abytes[r], lo[r], cnt[r]);
    for (uint32_t q = 0; q < m; ++q)
        snp_storage_window(S, nS, accts + 32 * first[q], first[q + 1] - first[q], sorigin + 32ull * q, slimit + 32ull * q, sbytes[q],
                           &lo[n + first[q]], &run[first[q]], &cnt[n + first[q]]);
    std::vector<uint64_t> coff(nseg + 1, 0);
    for (uint64_t r = 0; r < nseg; ++r) coff[r + 1] = coff[r] + cnt[r];
    const uint64_t C = coff[nseg];
    std::vector<uint64_t> x(C + 1, 0);
    for (uint64_t j = 0; j < C; ++j) {
        const uint64_t r = rg_segment(coff.data(), nseg, j), row = lo[r] + (j - coff[r]);
        const uint32_t len = r < n ? snp_slim(arena + krows[row].off, krows[row].len, nullptr) : snp_slot_body(S[row].val, nullptr);
        if (r < n && !len) return 1;
        x[j + 1] = x[j] + 32 + len;
    }
    for (uint32_t r = 0; r < n; ++r) ent[r] = snp_account_cut(&x[coff[r]], cnt[r], abytes[r]);
    for (uint32_t q = 0; q < m; ++q) {
        bool set = false;
        for (int b = 0; b < 32; ++b) set |= sorigin[32ull * q + b] != 0;
        const uint64_t R = n + first[q];
        const SnpServe sv = snp_storage_cut(&x[coff[R]], &cnt[R], &run[first[q]], first[q + 1] - first[q], set, sbytes[q], &ent[R]);
        served[q] = sv.served;
        proved[q] = sv.proved;
    }
    uint64_t e = 0, b = 0;
    for (uint64_t r = 0; r < nseg; ++r)
        for (uint64_t t = 0; t < ent[r]; ++t, ++e) {
            const uint64_t row = lo[r] + t, len = x[coff[r] + t + 1] - x[coff[r] + t] - 32;
            if (e >= cap || b + len > bcap) return 2;
            memcpy(keys + 32 * e, r < n ? krows[row].key : S[row].skey, 32);
            boff[e] = b;
            if (r < n) snp_slim(arena + krows[row].off, krows[row].len, bodies + b);
            else snp_slot_body(S[row].val, bodies + b);
            b += len;
        }
    boff[e] = b;
    return 0;
}
