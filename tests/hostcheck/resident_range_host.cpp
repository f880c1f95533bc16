// Test-only: compiles the DEVICE range statements of the resident world state (phant_b200/csrc/resident_range.cuh, on top of
// resident_read.cuh) as HOST code -- CUDA qualifiers and intrinsics defined away below, as in resident_read_host.cpp -- and
// runs one whole range call the way rs_range in trie.cu runs it: the parts of every range, the candidates, a sort by (range,
// key) (std::stable_sort in place of the device radix sort), duplicates dropped, resolution, ranks, selection and the fill.
// Built as a shared object by tests/test_resident_range_header_host.py; nothing in the product links or loads this.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <numeric>
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
#include "resident_range.cuh"

using namespace phant;

// the row layouts of trie.cu
struct alignas(16) KRow { uint8_t key[32]; uint64_t off; uint32_t len; uint8_t cache[33]; };
struct alignas(16) SlotRow { uint8_t akey[32], skey[32], val[32]; };
static_assert(sizeof(KRow) == 80 && sizeof(SlotRow) == 96, "row layout");

static std::vector<uint64_t> exclusive_scan(const std::vector<uint64_t>& v)
{
    std::vector<uint64_t> o(v.size() + 1, 0);
    for (size_t i = 0; i < v.size(); ++i) o[i + 1] = o[i] + v[i];
    return o;
}

// One range call: n account ranges, then m storage ranges (origin, limit: (n + m) x 32; sacct: m x 32; max: n + m) at the root
// `back` records ago.  Out: first (n + m + 1 entry offsets, account entries first), more (n + m), cands (n + m: the
// candidates each range had), and per entry e < cap its key (32 B) and value: nonce and balance | storageRoot | codeHash
// (96 B) for an account, the 32-byte value for a slot.  Returns 0, 1 when an entry did not resolve as present, 2 when the
// entries exceed cap.
extern "C" int hr_range(const KRow* krows, uint32_t nK, const uint8_t* arena, const SlotRow* S, uint32_t nS, const RdRec* recs, uint32_t back,
                        uint32_t n, uint32_t m, const uint8_t* origin, const uint8_t* limit, const uint8_t* sacct, const uint32_t* max, uint64_t cap,
                        uint64_t* first, uint8_t* more, uint64_t* cands, uint8_t* keys, uint64_t* nonce, uint8_t* acc96, uint8_t* val32)
{
    const uint32_t nr = n + m;
    const uint64_t P = back + 1, parts = P * nr;
    std::vector<uint32_t> lo(parts);
    std::vector<uint64_t> cnt(parts);
    for (uint32_t r = 0; r < nr; ++r) {
        if (r < n) rg_account_parts(recs, back, krows, nK, origin + 32ull * r, limit + 32ull * r, max[r], &lo[P * r], &cnt[P * r]);
        else rg_slot_parts(recs, back, S, nS, sacct + 32ull * (r - n), origin + 32ull * r, limit + 32ull * r, max[r], &lo[P * r], &cnt[P * r]);
    }
    const std::vector<uint64_t> poff = exclusive_scan(cnt);
    const uint64_t C = poff[parts];
    std::vector<uint8_t> ckeys;
    std::vector<uint32_t> cseg, perm;
    std::vector<uint64_t> x;
    if (back) {
        ckeys.resize(32 * C + 32);
        cseg.resize(C);
        for (uint64_t j = 0; j < C; ++j) {
            const uint64_t pp = rg_segment(poff.data(), parts, j);
            const uint32_t r = (uint32_t)(pp / P), p = (uint32_t)(pp % P);
            const uint8_t* k = r < n ? rg_account_key(recs, krows, p, lo[pp], j - poff[pp]) : rg_slot_key(recs, S, p, lo[pp], j - poff[pp]);
            memcpy(&ckeys[32 * j], k, 32);
            cseg[j] = r;
        }
        perm.resize(C);
        std::iota(perm.begin(), perm.end(), 0u);
        std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) {
            if (cseg[a] != cseg[b]) return cseg[a] < cseg[b];
            return memcmp(&ckeys[32ull * a], &ckeys[32ull * b], 32) < 0;
        });
        std::vector<uint64_t> pres(C);
        for (uint64_t j = 0; j < C; ++j) {
            const uint32_t i = perm[j], r = cseg[i];
            const uint8_t* key = &ckeys[32ull * i];
            if (j && cseg[perm[j - 1]] == r && rd_cmp32(&ckeys[32ull * perm[j - 1]], key) == 0) { pres[j] = 0; continue; }
            const uint32_t status = r < n ? rd_account(recs, back, krows, nK, arena, key).status : rd_slot(recs, back, S, nS, sacct + 32ull * (r - n), key).status;
            pres[j] = status == RD_PRESENT;
        }
        x = exclusive_scan(pres);
    }
    std::vector<uint64_t> ent(nr);
    for (uint32_t r = 0; r < nr; ++r) {
        const uint64_t present = back ? x[poff[P * (r + 1)]] - x[poff[P * r]] : cnt[r];
        rg_select(present, max[r], ent[r], more[r]);
        cands[r] = poff[P * (r + 1)] - poff[P * r];
    }
    const std::vector<uint64_t> E = exclusive_scan(ent);
    for (uint32_t r = 0; r <= nr; ++r) first[r] = E[r];
    if (E[nr] > cap) return 2;
    for (uint64_t e = 0; e < E[nr]; ++e) {
        const uint32_t r = (uint32_t)rg_segment(E.data(), nr, e);
        const uint64_t at = e - E[r];
        const uint8_t* key;
        if (back) key = &ckeys[32ull * perm[rg_nth_present(x.data(), poff[P * r], poff[P * (r + 1)], at)]];
        else key = r < n ? rg_account_key(recs, krows, 0, lo[r], at) : rg_slot_key(recs, S, 0, lo[r], at);
        memcpy(keys + 32 * e, key, 32);
        if (r < n) {
            const RdAccount a = rd_account(recs, back, krows, nK, arena, key);
            if (a.status != RD_PRESENT) return 1;
            nonce[e] = a.nonce;
            for (uint32_t b = 0; b < 32; ++b) {
                acc96[96 * e + b] = b >= 32 - a.bal_len ? a.bal[b - (32 - a.bal_len)] : 0;
                acc96[96 * e + 32 + b] = a.sroot[b];
                acc96[96 * e + 64 + b] = a.code[b];
            }
        } else {
            const RdSlot v = rd_slot(recs, back, S, nS, sacct + 32ull * (r - n), key);
            if (v.status != RD_PRESENT) return 1;
            memcpy(val32 + 32 * e, v.val, 32);
        }
    }
    return 0;
}
