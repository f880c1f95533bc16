// trie.cu -- trie builders on the device: M (== mptize), S (state root), U (resident complete trie).
//
// M restates src/mpt/mpt.zig:38-314 as a level-synchronous FOREST builder over sorted keys:
//   top-down   every (extension+)branch unit is a key range [lo, hi) of the sorted list; its branch depth is the
//              common prefix of the range (mpt.zig:83-106), a key that ends there is the branch value
//              (mpt.zig:65-69), and the 16 children are found by binary search on the next nibble
//              (mpt.zig:72-79) -- 16 threads per unit, one BFS level per launch;
//   bottom-up  leaves first, then unit levels deepest-first: RLP is written into a scratch arena
//              (leaf mpt.zig:255-281, branch :218-247, extension :180-209, hex-prefix :285-314) and hashed by
//              the SAME batched Keccak kernel the verifier uses; a child enters its parent as raw RLP when
//              < 32 bytes, else as its hash (mpt.zig:104,112); the root is always hashed (mpt.zig:42).
// A forest (many tries at once) is what S needs: all storage tries of a state are built together.
// S follows evmone/test/state/mpt_hash.cpp:15-36 for the trie contents (phant has no StateDB.root()).
// U is the dirty-frontier recompute over a resident complete 16-ary trie (BASELINE.json config C4).
#include "../../include/phant_gpu.h"
#include "common.cuh"
#include "ctx.cuh"
#include "keccak_f1600.cuh"

#include <chrono>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <string.h>
#include <algorithm>
#include <deque>
#include <new>
#include <vector>

using namespace phant;

#define CU(expr)                                                                \
    do {                                                                        \
        cudaError_t e_ = (expr);                                                \
        if (e_ != cudaSuccess) return ctx->fail(e_, #expr, __FILE__, __LINE__); \
    } while (0)
#define RC(expr)                  \
    do {                          \
        int rc_ = (expr);         \
        if (rc_ != 0) return rc_; \
    } while (0)

// Witness output (phant_gpu_resident_state_witness): nodes appended in any order, each with its digest; an append past a
// capacity is counted but not written, so the caller sees what it needs and runs again
struct WNode { uint64_t off; uint32_t len, pad; };
struct WitnessOut {
    uint8_t* bytes; uint64_t cap_bytes;
    WNode* nodes; uint8_t* digests; uint64_t cap_nodes;
    unsigned long long* used; // [0] nodes, [1] bytes
};
// build_forest's export: the nodes of every segment on the path of some proof key of its trie (32-byte keys only)
struct ForestExport {
    const uint8_t* pkeys;      // proof keys, 32 bytes each, sorted by (trie, key)
    const uint32_t* ptrie;     // the trie of each
    uint32_t np;
    const uint32_t* seg_trie;  // the trie of each forest segment
    const uint32_t* seg_of_key;
    WitnessOut out;
};

namespace {

// development knob PHANT_GPU_TRACE=1: wall time of the phases of a sparse-trie update on stderr (adds a synchronisation per phase)
struct PhaseTrace {
    cudaStream_t s;
    bool on;
    std::chrono::steady_clock::time_point t0;
    explicit PhaseTrace(cudaStream_t st) : s(st)
    {
        static int env = -1;
        if (env < 0) { const char* e = getenv("PHANT_GPU_TRACE"); env = e && *e == '1'; }
        on = env == 1;
        if (on) { cudaStreamSynchronize(s); t0 = std::chrono::steady_clock::now(); }
    }
    void mark(const char* what)
    {
        if (!on) return;
        cudaStreamSynchronize(s);
        const auto t1 = std::chrono::steady_clock::now();
        fprintf(stderr, "[phant trace] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
        t0 = t1;
    }
};


constexpr uint32_t NONE = 0xffffffffu;
constexpr uint32_t KIND_LEAF = 1u << 30, KIND_NODE = 2u << 30, KIND_MASK = 3u << 30, IDX_MASK = ~KIND_MASK;

__constant__ uint8_t EMPTY_ROOT_D[32] = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45,
                                         0xe6, 0x92, 0xc0, 0xf8, 0x6e, 0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c,
                                         0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};
constexpr uint8_t EMPTY_ROOT_H[32] = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                      0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};

// ---------------------------------------------------------------- RLP helpers (device)
__device__ __forceinline__ uint32_t be_len(uint64_t v)
{
    uint32_t n = 0;
    while (v) { ++n; v >>= 8; }
    return n;
}
__device__ __forceinline__ uint64_t str_size(uint64_t len, uint32_t first_byte)
{
    if (len == 1 && first_byte < 0x80) return 1;
    if (len <= 55) return 1 + len;
    return 1 + be_len(len) + len;
}
__device__ __forceinline__ uint32_t hdr_size(uint64_t payload) { return payload <= 55 ? 1 : 1 + be_len(payload); }
__device__ __forceinline__ uint32_t put_hdr(uint8_t* out, uint64_t len, uint32_t short_base, uint32_t long_base)
{
    if (len <= 55) { out[0] = (uint8_t)(short_base + len); return 1; }
    const uint32_t n = be_len(len);
    out[0] = (uint8_t)(long_base + n);
    for (uint32_t i = 0; i < n; ++i) out[1 + i] = (uint8_t)(len >> (8 * (n - 1 - i)));
    return 1 + n;
}

// ---------------------------------------------------------------- key access
struct Keys {
    const uint8_t* bytes;
    const uint32_t* off; // n+1
};
__device__ __forceinline__ uint32_t nlen(const Keys& k, uint32_t i) { return 2 * (k.off[i + 1] - k.off[i]); }
__device__ __forceinline__ uint32_t nib(const Keys& k, uint32_t i, uint32_t pos)
{
    const uint8_t b = k.bytes[k.off[i] + (pos >> 1)];
    return (pos & 1) ? (b & 15u) : (b >> 4);
}
// common prefix of keys i and j in nibbles
__device__ uint32_t lcp(const Keys& k, uint32_t i, uint32_t j)
{
    const uint32_t li = k.off[i + 1] - k.off[i], lj = k.off[j + 1] - k.off[j];
    const uint32_t m = li < lj ? li : lj;
    const uint8_t* a = k.bytes + k.off[i];
    const uint8_t* b = k.bytes + k.off[j];
    uint32_t t = 0;
    while (t < m && a[t] == b[t]) ++t;
    if (t == m) return 2 * m;
    return 2 * t + (((a[t] ^ b[t]) & 0xf0) ? 0 : 1);
}
// hex-prefix bytes of nibbles [from, to) of key i (mpt.zig:285-314); returns count
__device__ uint32_t hp_size(uint32_t cnt) { return 1 + cnt / 2; }
__device__ uint32_t put_hp(uint8_t* out, const Keys& k, uint32_t i, uint32_t from, uint32_t to, bool leaf)
{
    const uint32_t cnt = to - from;
    uint32_t o = 0, q = from;
    if (cnt & 1) { out[o++] = (uint8_t)(((leaf ? 3 : 1) << 4) | nib(k, i, q)); ++q; }
    else out[o++] = (uint8_t)((leaf ? 2 : 0) << 4);
    for (; q < to; q += 2) out[o++] = (uint8_t)((nib(k, i, q) << 4) | nib(k, i, q + 1));
    return o;
}
__device__ uint32_t hp_first_byte(const Keys& k, uint32_t i, uint32_t from, uint32_t to, bool leaf)
{
    const uint32_t cnt = to - from;
    return (cnt & 1) ? (((leaf ? 3u : 1u) << 4) | nib(k, i, from)) : ((leaf ? 2u : 0u) << 4);
}

// ---------------------------------------------------------------- node tables
struct Tables {
    // per unit (capacity = n_keys)
    uint32_t *lo, *hi, *ext_from, *depth, *child; // child[16 * id + v]
    uint8_t* has_value;
    uint32_t* ext_list; // per level: ids of units with an extension, at the level's base
    // per key
    uint32_t* leaf_start; // nibble where the leaf path starts; NONE for branch-value keys
    // references (what a parent copies): 33 bytes + length, for leaves [0, n) and units [n, n + cap)
    uint8_t* ref;
    uint8_t* ref_len;
    uint8_t* top_digest; // per unit: hash of its topmost encoding (extension if any, else branch)
    // per segment
    uint32_t* seg_root; // KIND | idx, or 0 = empty
};

// ---------------------------------------------------------------- validation
__global__ void check_sorted_kernel(Keys k, const uint64_t* __restrict__ val_off, const uint32_t* __restrict__ seg_of_key, uint32_t n,
                                    uint32_t* flags /*[0] unsorted, [1] some key is a prefix of its successor, [2] max key bytes, [3] max value bytes*/)
{
    uint32_t max_k = 0, max_v = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t la = k.off[i + 1] - k.off[i];
        const uint64_t lv = val_off[i + 1] - val_off[i];
        max_k = la > max_k ? la : max_k;
        const uint32_t lv32 = lv > 0xffffffffull ? 0xffffffffu : (uint32_t)lv;
        max_v = lv32 > max_v ? lv32 : max_v;
        if (i + 1 >= n || (seg_of_key && seg_of_key[i] != seg_of_key[i + 1])) continue;
        const uint32_t lb = k.off[i + 2] - k.off[i + 1];
        const uint8_t* a = k.bytes + k.off[i];
        const uint8_t* b = k.bytes + k.off[i + 1];
        const uint32_t m = la < lb ? la : lb;
        uint32_t t = 0;
        while (t < m && a[t] == b[t]) ++t;
        const bool ok = t < m ? a[t] < b[t] : la < lb; // strictly increasing; a strict prefix sorts first
        if (!ok) atomicExch(&flags[0], 1u);
        if (t == la) atomicExch(&flags[1], 1u);        // key i is a prefix of key i+1: that branch will carry a value
    }
    for (int o = 16; o; o >>= 1) {
        const uint32_t ok = __shfl_down_sync(0xffffffffu, max_k, o), ov = __shfl_down_sync(0xffffffffu, max_v, o);
        max_k = ok > max_k ? ok : max_k;
        max_v = ov > max_v ? ov : max_v;
    }
    if ((threadIdx.x & 31) == 0) { atomicMax(&flags[2], max_k); atomicMax(&flags[3], max_v); }
}

// ---------------------------------------------------------------- top-down
__global__ void init_roots_kernel(const uint32_t* __restrict__ seg_off, uint32_t n_seg, Tables t, uint32_t* counters /*[0]=units*/,
                                  uint32_t start_all /*nibbles already consumed above each segment's root (0 for a whole trie)*/,
                                  const uint32_t* __restrict__ seg_start /*nullable: the same per segment*/)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
        const uint32_t lo = seg_off[s], hi = seg_off[s + 1], start = seg_start ? seg_start[s] : start_all;
        if (hi == lo) { t.seg_root[s] = 0; continue; }
        if (hi - lo == 1) { t.seg_root[s] = KIND_LEAF | lo; t.leaf_start[lo] = start; continue; }
        const uint32_t id = atomicAdd(&counters[0], 1u);
        t.lo[id] = lo; t.hi[id] = hi; t.ext_from[id] = start;
        t.seg_root[s] = KIND_NODE | id;
    }
}

// One branch unit, 16 cooperating lanes (lane v looks after child nibble v): find the branch depth, the branch value and
// the 16 child ranges; children with >= 2 keys become units of the next level (appended at next_base + counter).
__device__ __forceinline__ void expand_unit(const Keys& k, const Tables& t, uint32_t id, uint32_t v, uint32_t sub, uint32_t next_base,
                                            uint32_t* next_count, uint32_t* ext_count, uint32_t ext_base)
{
    const uint32_t lo = t.lo[id], hi = t.hi[id], from = t.ext_from[id];
    uint32_t p = 0;
    if (v == 0) {
        p = lcp(k, lo, hi - 1);
        const uint32_t l0 = nlen(k, lo);
        if (l0 < p) p = l0;
    }
    p = __shfl_sync(sub, p, 0, 16);
    const bool has_value = nlen(k, lo) == p;
    const uint32_t first = lo + (has_value ? 1 : 0);
    // lower bound of nibble value v at depth p within [first, hi)
    uint32_t a = first, b = hi;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (nib(k, mid, p) < v) a = mid + 1; else b = mid;
    }
    uint32_t ub = __shfl_down_sync(sub, a, 1, 16);
    if (v == 15) ub = hi;
    uint32_t child = 0;
    const uint32_t c = ub - a;
    if (c == 1) {
        child = KIND_LEAF | a;
        t.leaf_start[a] = p + 1;
    } else if (c >= 2) {
        const uint32_t nid = next_base + atomicAdd(next_count, 1u);
        t.lo[nid] = a; t.hi[nid] = ub; t.ext_from[nid] = p + 1;
        child = KIND_NODE | nid;
    }
    t.child[16 * id + v] = child;
    if (v == 0) {
        t.depth[id] = p;
        t.has_value[id] = has_value ? 1 : 0;
        if (has_value) t.leaf_start[lo] = NONE;
        if (p > from) t.ext_list[ext_base + atomicAdd(ext_count, 1u)] = id;
    }
}

// one BFS level per launch (large tries)
__global__ void __launch_bounds__(128)
expand_kernel(Keys k, Tables t, uint32_t beg, uint32_t cnt, uint32_t next_base, uint32_t* counters /*[1]=next units, [2]=ext in this level*/)
{
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t sub = 0xffffu << (threadIdx.x & 16); // my half-warp
    for (uint32_t u = gid >> 4; u < cnt; u += (gridDim.x * blockDim.x) >> 4) // the 16 lanes of a half-warp share u
        expand_unit(k, t, beg + u, threadIdx.x & 15, sub, next_base, &counters[1], &counters[2], beg);
}

// the whole BFS in ONE launch of one CTA (small tries are launch-bound): levels[0] = number of levels, then
// (begin, count, extensions) per level; stops at max_levels (the caller sizes it from the key length)
__global__ void __launch_bounds__(1024)
bfs_small_kernel(Keys k, Tables t, uint32_t first_cnt, uint32_t max_levels, uint32_t* __restrict__ levels)
{
    __shared__ uint32_t s_next, s_ext;
    const uint32_t sub = 0xffffu << (threadIdx.x & 16);
    uint32_t beg = 0, cnt = first_cnt, nl = 0;
    while (cnt && nl < max_levels) {
        if (threadIdx.x == 0) { s_next = 0; s_ext = 0; }
        __syncthreads();
        for (uint32_t u = threadIdx.x >> 4; u < cnt; u += blockDim.x >> 4)
            expand_unit(k, t, beg + u, threadIdx.x & 15, sub, beg + cnt, &s_next, &s_ext, beg);
        __syncthreads();
        if (threadIdx.x == 0) { levels[1 + 3 * nl] = beg; levels[2 + 3 * nl] = cnt; levels[3 + 3 * nl] = s_ext; }
        beg += cnt;
        cnt = s_next;
        ++nl;
        __syncthreads();
    }
    if (threadIdx.x == 0) { levels[0] = nl; levels[1 + 3 * max_levels] = cnt; } // cnt != 0: deeper than max_levels (never with max_levels >= key nibbles)
}

// ---------------------------------------------------------------- leaves
struct Vals {
    const uint8_t* bytes;
    const uint64_t* off;
};

// ids (nullable): work item j is key ids[j] (the leaves that still have to be encoded when a leaf-reference cache is in use)
__global__ void leaf_size_kernel(Keys k, Vals vals, Tables t, uint32_t n, uint64_t* __restrict__ size, const uint32_t* __restrict__ ids)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t i = ids ? ids[j] : j;
        const uint32_t ls = t.leaf_start[i];
        uint64_t sz = 0;
        if (ls != NONE) {
            const uint32_t nl = nlen(k, i);
            const uint32_t hpn = hp_size(nl - ls);
            const uint64_t vl = vals.off[i + 1] - vals.off[i];
            const uint64_t payload = str_size(hpn, hp_first_byte(k, i, ls, nl, true)) + str_size(vl, vl ? vals.bytes[vals.off[i]] : 0);
            sz = hdr_size(payload) + payload;
        }
        size[j] = sz;
    }
}
// one warp per leaf: lane 0 writes the headers and the path, all lanes copy the value
__global__ void __launch_bounds__(256)
leaf_encode_kernel(Keys k, Vals vals, Tables t, uint32_t n, const uint64_t* __restrict__ aoff, uint8_t* __restrict__ arena,
                   uint64_t* __restrict__ size_out /*nullable: slot layout, the encoder reports the sizes itself*/,
                   const uint32_t* __restrict__ ids /*nullable: work item j is key ids[j]*/)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t i = ids ? ids[j] : j;
        const uint32_t ls = t.leaf_start[i];
        if (ls == NONE) { if (size_out && lane == 0) size_out[j] = 0; continue; }
        uint8_t* out = arena + aoff[j];
        const uint32_t nl = nlen(k, i);
        const uint32_t hpn = hp_size(nl - ls);
        const uint64_t vl = vals.off[i + 1] - vals.off[i];
        const uint8_t* v = vals.bytes + vals.off[i];
        const uint32_t hp0 = hp_first_byte(k, i, ls, nl, true);
        const uint64_t s_hp = str_size(hpn, hp0), s_v = str_size(vl, vl ? v[0] : 0);
        const uint32_t h = hdr_size(s_hp + s_v);
        if (lane == 0) {
            if (size_out) size_out[j] = h + s_hp + s_v;
            put_hdr(out, s_hp + s_v, 0xc0, 0xf7);
            uint8_t* q = out + h;
            if (s_hp > hpn) q += put_hdr(q, hpn, 0x80, 0xb7);
            put_hp(q, k, i, ls, nl, true);
            q = out + h + s_hp;
            if (s_v > vl) put_hdr(q, vl, 0x80, 0xb7);
        }
        uint8_t* dst = out + h + s_hp + (s_v - vl);
        for (uint64_t b = lane; b < vl; b += 32) dst[b] = v[b];
    }
}
// Leaf-reference cache (resident tries): row i = [leaf_start + 1 (0 = nothing cached)] + the 32-byte digest of key i's leaf as
// it was last encoded.  A leaf's encoding depends on (key, the nibble its path starts at, value) only, so a row whose depth
// byte matches needs neither encode nor hash: its reference is written here and the key is left out of the to-do list.
__global__ void leaf_cache_probe_kernel(Tables t, uint32_t n, const uint8_t* __restrict__ cache, uint8_t* __restrict__ leaf_digests,
                                        uint32_t* __restrict__ todo_flag)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t ls = t.leaf_start[i];
        const uint8_t* row = cache + 33ull * i;
        const bool hit = ls != NONE && ls < 255 && row[0] == (uint8_t)(ls + 1);
        todo_flag[i] = hit ? 0 : 1;
        if (hit) {
            uint8_t* r = t.ref + 33ull * i;
            r[0] = 0xa0;
            for (uint32_t b = 0; b < 32; ++b) { r[1 + b] = row[1 + b]; leaf_digests[32ull * i + b] = row[1 + b]; }
            t.ref_len[i] = 33;
        }
    }
}
__global__ void leaf_cache_store_kernel(Tables t, uint32_t n, const uint8_t* __restrict__ leaf_digests, uint8_t* __restrict__ cache_out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t ls = t.leaf_start[i];
        uint8_t* row = cache_out + 33ull * i;
        const bool hashed = ls != NONE && ls < 255 && t.ref_len[i] == 33; // embedded leaves (< 32 bytes) are never cached
        row[0] = hashed ? (uint8_t)(ls + 1) : 0;
        if (hashed)
            for (uint32_t b = 0; b < 32; ++b) row[1 + b] = leaf_digests[32ull * i + b];
    }
}
__global__ void compact_iota_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, uint32_t n, uint32_t* __restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (flag[i]) out[pos[i]] = i;
}
// reference of item j (leaf or encoded unit): raw RLP when < 32 bytes, else 0xa0 || digest
__global__ void finalize_ref_kernel(uint32_t cnt, const uint32_t* __restrict__ ids /*nullable: identity*/, uint32_t id_base,
                                    const uint64_t* __restrict__ aoff, const uint64_t* __restrict__ alen /*nullable: CSR*/,
                                    const uint8_t* __restrict__ arena,
                                    const uint8_t* __restrict__ digests, uint32_t ref_base, Tables t, uint8_t* __restrict__ top_digest)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        const uint32_t id = ids ? ids[j] : id_base + j;
        const uint64_t len = alen ? alen[j] : aoff[j + 1] - aoff[j];
        uint8_t* r = t.ref + 33ull * (ref_base + id);
        if (len == 0) { t.ref_len[ref_base + id] = 0; continue; } // not a leaf (branch-value key)
        if (len < 32) {
            for (uint32_t b = 0; b < len; ++b) r[b] = arena[aoff[j] + b];
            t.ref_len[ref_base + id] = (uint8_t)len;
        } else {
            r[0] = 0xa0;
            for (uint32_t b = 0; b < 32; ++b) r[1 + b] = digests[32ull * j + b];
            t.ref_len[ref_base + id] = 33;
        }
        if (top_digest)
            for (uint32_t b = 0; b < 32; ++b) top_digest[32ull * id + b] = digests[32ull * j + b];
    }
}

// ---------------------------------------------------------------- branches and extensions
__device__ __forceinline__ uint32_t child_ref_index(uint32_t child, uint32_t n_keys)
{
    return (child & KIND_MASK) == KIND_LEAF ? (child & IDX_MASK) : n_keys + (child & IDX_MASK);
}
__global__ void branch_size_kernel(Keys k, Vals vals, Tables t, uint32_t n_keys, uint32_t beg, uint32_t cnt, uint64_t* __restrict__ size)
{
    for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < cnt; u += gridDim.x * blockDim.x) {
        const uint32_t id = beg + u;
        uint64_t payload = 0;
        for (uint32_t v = 0; v < 16; ++v) {
            const uint32_t c = t.child[16 * id + v];
            payload += c ? t.ref_len[child_ref_index(c, n_keys)] : 1;
        }
        if (t.has_value[id]) {
            const uint32_t i = t.lo[id];
            const uint64_t vl = vals.off[i + 1] - vals.off[i];
            payload += str_size(vl, vl ? vals.bytes[vals.off[i]] : 0);
        } else payload += 1;
        size[u] = hdr_size(payload) + payload;
    }
}
// one warp per unit: lane v < 16 places child v at the prefix sum of the reference sizes, all lanes copy the value
__global__ void __launch_bounds__(256)
branch_encode_kernel(Keys k, Vals vals, Tables t, uint32_t n_keys, uint32_t beg, uint32_t cnt, const uint64_t* __restrict__ aoff,
                     uint64_t* __restrict__ alen /*nullable: CSR*/, bool self_size /*slot layout: compute and store alen here*/,
                     uint8_t* __restrict__ arena)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < cnt; u += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t id = beg + u;
        uint8_t* out = arena + aoff[u];
        uint64_t total = self_size ? 0 : (alen ? alen[u] : aoff[u + 1] - aoff[u]);
        uint32_t c = 0, sz = 0, ri = 0;
        if (lane < 16) {
            c = t.child[16 * id + lane];
            if (c) { ri = child_ref_index(c, n_keys); sz = t.ref_len[ri]; } else sz = 1;
        }
        uint32_t pre = sz; // inclusive scan over lanes 0..15
        for (int o = 1; o < 16; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= (uint32_t)o) pre += y;
        }
        const uint32_t refs_total = __shfl_sync(0xffffffffu, pre, 15);
        const uint64_t payload_wo_value = refs_total;
        if (self_size) {
            uint64_t s_val = 1;
            if (t.has_value[id]) {
                const uint32_t i = t.lo[id];
                const uint64_t vl = vals.off[i + 1] - vals.off[i];
                s_val = str_size(vl, vl ? vals.bytes[vals.off[i]] : 0);
            }
            total = hdr_size(refs_total + s_val) + refs_total + s_val;
            if (lane == 0) alen[u] = total;
        }
        // total = header + payload: the header size (1..5) is the one consistent with the payload it leaves
        uint32_t hdr = 1;
        for (uint32_t cand = 1; cand <= 5; ++cand) {
            const uint64_t pay = total - cand;
            if (hdr_size(pay) == cand) { hdr = cand; break; }
        }
        if (lane == 0) put_hdr(out, total - hdr, 0xc0, 0xf7);
        if (lane < 16) {
            uint8_t* q = out + hdr + (pre - sz);
            if (c) {
                const uint8_t* r = t.ref + 33ull * ri;
                for (uint32_t b = 0; b < sz; ++b) q[b] = r[b];
            } else q[0] = 0x80;
        }
        uint8_t* q = out + hdr + payload_wo_value;
        if (t.has_value[id]) {
            const uint32_t i = t.lo[id];
            const uint64_t vl = vals.off[i + 1] - vals.off[i];
            const uint8_t* v = vals.bytes + vals.off[i];
            const uint64_t s_v = str_size(vl, vl ? v[0] : 0);
            if (lane == 0 && s_v > vl) put_hdr(q, vl, 0x80, 0xb7);
            uint8_t* dst = q + (s_v - vl);
            for (uint64_t b = lane; b < vl; b += 32) dst[b] = v[b];
        } else if (lane == 0) q[0] = 0x80;
    }
}
__global__ void ext_size_kernel(Keys k, Tables t, uint32_t n_keys, const uint32_t* __restrict__ ids, uint32_t cnt, uint64_t* __restrict__ size)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        const uint32_t id = ids[j];
        const uint32_t from = t.ext_from[id], to = t.depth[id], i = t.lo[id];
        const uint32_t hpn = hp_size(to - from);
        const uint64_t payload = str_size(hpn, hp_first_byte(k, i, from, to, false)) + t.ref_len[n_keys + id];
        size[j] = hdr_size(payload) + payload;
    }
}
__global__ void ext_encode_kernel(Keys k, Tables t, uint32_t n_keys, const uint32_t* __restrict__ ids, uint32_t cnt,
                                  const uint64_t* __restrict__ aoff, uint8_t* __restrict__ arena, uint64_t* __restrict__ size_out /*nullable*/)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        const uint32_t id = ids[j];
        const uint32_t from = t.ext_from[id], to = t.depth[id], i = t.lo[id];
        const uint32_t hpn = hp_size(to - from);
        const uint64_t s_hp = str_size(hpn, hp_first_byte(k, i, from, to, false));
        const uint32_t rl = t.ref_len[n_keys + id];
        uint8_t* out = arena + aoff[j];
        if (size_out) size_out[j] = hdr_size(s_hp + rl) + s_hp + rl;
        uint8_t* q = out + put_hdr(out, s_hp + rl, 0xc0, 0xf7);
        if (s_hp > hpn) q += put_hdr(q, hpn, 0x80, 0xb7);
        q += put_hp(q, k, i, from, to, false);
        const uint8_t* r = t.ref + 33ull * (n_keys + id);
        for (uint32_t b = 0; b < rl; ++b) q[b] = r[b];
    }
}
__global__ void gather_roots_kernel(Tables t, uint32_t n_seg, const uint8_t* __restrict__ leaf_digests, uint8_t* __restrict__ roots)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
        const uint32_t r = t.seg_root[s];
        const uint8_t* src = EMPTY_ROOT_D;
        if ((r & KIND_MASK) == KIND_LEAF) src = leaf_digests + 32ull * (r & IDX_MASK);
        else if ((r & KIND_MASK) == KIND_NODE) src = t.top_digest + 32ull * (r & IDX_MASK);
        for (uint32_t b = 0; b < 32; ++b) roots[32ull * s + b] = src[b];
    }
}

// ---------------------------------------------------------------- witness export
// room for one node of len bytes in the witness output (nullptr past a capacity), its digest written
__device__ uint8_t* wit_reserve(const WitnessOut& o, uint32_t len, const uint8_t* digest)
{
    const unsigned long long i = atomicAdd(&o.used[0], 1ull), off = atomicAdd(&o.used[1], (unsigned long long)len);
    if (i >= o.cap_nodes || off + len > o.cap_bytes) return nullptr;
    o.nodes[i] = WNode{off, len, 0};
    for (uint32_t b = 0; b < 32; ++b) o.digests[32 * i + b] = digest[b];
    return o.bytes + off;
}
__device__ __forceinline__ uint32_t lcp_nib32(const uint8_t* a, const uint8_t* b)
{
    uint32_t t = 0;
    while (t < 32 && a[t] == b[t]) ++t;
    return t == 32 ? 64 : 2 * t + (((a[t] ^ b[t]) & 0xf0) ? 0 : 1);
}
// whether the first d nibbles of `key` start some proof key of `trie` (the proof keys with that prefix are contiguous, so the
// two around the lower bound of (trie, key) decide)
__device__ bool on_proof_path(const ForestExport& x, uint32_t trie, const uint8_t* key, uint32_t d)
{
    uint32_t a = 0, b = x.np;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        bool less = x.ptrie[mid] < trie;
        if (x.ptrie[mid] == trie) {
            const uint8_t* p = x.pkeys + 32ull * mid;
            uint32_t t = 0;
            while (t < 32 && p[t] == key[t]) ++t;
            less = t < 32 && p[t] < key[t];
        }
        if (less) a = mid + 1; else b = mid;
    }
    for (uint32_t j = a ? a - 1 : 0; j <= a && j < x.np; ++j)
        if (x.ptrie[j] == trie && lcp_nib32(x.pkeys + 32ull * j, key) >= d) return true;
    return false;
}
// the nodes of one encode pass that a witness holds: on a proof key's path, and 32 bytes or more or the root of a whole trie.
// what: 0 leaves (item j is key ids[j], or j), 1 branch units (id beg + j), 2 extensions (id ids[j])
__global__ void forest_export_kernel(Keys k, Tables t, ForestExport x, uint32_t what, uint32_t cnt, const uint32_t* __restrict__ ids, uint32_t beg,
                                     const uint64_t* __restrict__ aoff, const uint64_t* __restrict__ alen /*nullable: CSR*/,
                                     const uint8_t* __restrict__ arena, const uint8_t* __restrict__ digests)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        uint32_t i, d;
        if (what == 0) {
            i = ids ? ids[j] : j;
            d = t.leaf_start[i];
            if (d == NONE) continue;
        } else {
            const uint32_t id = what == 1 ? beg + j : ids[j];
            i = t.lo[id];
            d = what == 1 ? t.depth[id] : t.ext_from[id];
        }
        const uint64_t len = alen ? alen[j] : aoff[j + 1] - aoff[j];
        if (len < 32 && d != 0) continue; // embedded in its parent
        if (!on_proof_path(x, x.seg_trie[x.seg_of_key[i]], k.bytes + k.off[i], d)) continue;
        uint8_t* dst = wit_reserve(x.out, (uint32_t)len, digests + 32ull * j);
        if (dst)
            for (uint64_t b = 0; b < len; ++b) dst[b] = arena[aoff[j] + b];
    }
}

__global__ void fixed_offsets_kernel(uint64_t* off, uint64_t n, uint64_t stride)
{
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (uint64_t)gridDim.x * blockDim.x) off[i] = stride * i;
}

unsigned grid1d(int device, uint64_t work_items, unsigned block, unsigned per_item = 1)
{
    uint64_t blocks = (work_items * per_item + block - 1) / block;
    const uint64_t cap = (uint64_t)keccak_num_sms(device) * 16;
    if (blocks > cap) blocks = cap;
    return (unsigned)(blocks ? blocks : 1);
}

// exclusive scan of cnt u32 items
int scan_u32(phant_gpu_ctx* ctx, const uint32_t* in, uint32_t* out, uint64_t cnt)
{
    return cub_call(ctx, [&](void* tmp, size_t& b) { return cub::DeviceScan::ExclusiveSum(tmp, b, in, out, (int64_t)cnt, ctx->stream); });
}
// exclusive scan of cnt u64 sizes into cnt+1 offsets (in[cnt] must be readable; it is forced to 0 first)
int scan_sizes(phant_gpu_ctx* ctx, uint64_t* sizes, uint64_t* offs, uint64_t cnt)
{
    CU(cudaMemsetAsync(sizes + cnt, 0, 8, ctx->stream));
    return cub_call(ctx, [&](void* tmp, size_t& b) {
        return cub::DeviceScan::ExclusiveSum(tmp, b, (const uint64_t*)sizes, offs, (int64_t)(cnt + 1), ctx->stream);
    });
}

// ------------------------------------------------------------------------------------------------
// forest builder: many tries at once over keys and values on the device, keys sorted inside each segment
// ------------------------------------------------------------------------------------------------
struct Forest {
    const uint8_t* keys = nullptr;
    const uint32_t* key_off = nullptr;    // n + 1
    const uint8_t* vals = nullptr;
    const uint64_t* val_off = nullptr;    // n + 1
    uint32_t n = 0;
    const uint32_t* seg_off = nullptr;    // n_seg + 1: segment s is keys [seg_off[s], seg_off[s + 1])
    uint32_t n_seg = 0;
    const uint32_t* seg_of_key = nullptr; // n: the sortedness check does not compare across segments (nullable: it does)
    uint8_t* roots = nullptr;             // n_seg x 32
    uint32_t slot_stride = 0;             // the slot layout with this leaf stride (no key a prefix of another); 0: chosen on the device
    uint32_t start_depth = 0;             // key nibbles consumed above every segment's root
    const uint32_t* seg_start = nullptr;  // n_seg: start depth per segment (nullable: start_depth for all)
    const uint8_t* leaf_cache = nullptr;  // n x 33: leaf references of an earlier build (resident tries), see leaf_cache_probe_kernel
    uint8_t* leaf_cache_out = nullptr;    // n x 33: the references of this build
    const ForestExport* xp = nullptr;     // copy out the nodes on given key paths
};

int build_forest(phant_gpu_ctx* ctx, const Forest& f)
{
    cudaStream_t s = ctx->stream;
    const int device = ctx->device;
    const uint32_t n = f.n, n_seg = f.n_seg;
    if (n_seg == 0) return PHANT_GPU_OK;
    PhaseTrace trf(s);
    const Keys k{f.keys, f.key_off};
    const Vals vals{f.vals, f.val_off};
    const uint32_t cap = n ? n : 1;
    constexpr uint32_t MAXL = 160; // levels of the single-CTA BFS: slot layout implies keys <= 64 bytes = 128 nibbles, 129 levels

    // what the key count sizes: the tables, counters, the single-CTA BFS's levels, and the leaves' digests, cache
    // compaction, sizes and offsets
    Tables t;
    uint32_t *counters, *bfs_levels, *cache_flag, *cache_pos, *cache_list;
    uint8_t *leaf_digests, *leaf_compact_digests;
    uint64_t *leaf_size, *leaf_off;
    const uint32_t n_cached = f.leaf_cache ? n + 2 : 0;
    RC(carve(ctx, ctx->fo_keys, [&](Carve& c) {
        t.lo = c.take<uint32_t>(cap); t.hi = c.take<uint32_t>(cap); t.ext_from = c.take<uint32_t>(cap); t.depth = c.take<uint32_t>(cap);
        t.child = c.take<uint32_t>(16ull * cap);
        t.has_value = c.take<uint8_t>(cap);
        t.ext_list = c.take<uint32_t>(cap); t.leaf_start = c.take<uint32_t>(cap); t.seg_root = c.take<uint32_t>(n_seg);
        t.ref = c.take<uint8_t>(33ull * 2 * cap); t.ref_len = c.take<uint8_t>(2ull * cap); t.top_digest = c.take<uint8_t>(32ull * cap);
        counters = c.take<uint32_t>(16);
        bfs_levels = c.take<uint32_t>(2 + 3 * MAXL);
        leaf_digests = c.take<uint8_t>(32ull * n);
        cache_flag = c.take<uint32_t>(n_cached); cache_pos = c.take<uint32_t>(n_cached); cache_list = c.take<uint32_t>(n_cached);
        leaf_compact_digests = c.take<uint8_t>(32ull * (f.leaf_cache ? n : 0));
        leaf_size = c.take<uint64_t>(n + 2); leaf_off = c.take<uint64_t>(n + 2);
    }));
    CU(cudaMemsetAsync(counters, 0, 64, s));
    CU(cudaMemsetAsync(t.leaf_start, 0xff, 4ull * cap, s));

    // keys must be strictly sorted inside each segment (mpt.zig:39 asserts)
    if (n) {
        check_sorted_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(k, f.val_off, f.seg_of_key, n, counters + 4);
        ctx->stats.launches++;
    }
    init_roots_kernel<<<grid1d(device, n_seg, 256), 256, 0, s>>>(f.seg_off, n_seg, t, counters, f.start_depth, f.seg_start);
    ctx->stats.launches++;
    uint32_t h[8];
    CU(cudaMemcpyAsync(h, counters, 32, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (h[4]) return PHANT_GPU_E_INVALID;
    // layout choice (see "Two arena layouts" below), from what the check kernel saw: slots need no branch values and small leaves
    uint32_t leaf_stride = 0;
    if (f.slot_stride) leaf_stride = f.slot_stride;
    else if (n && !h[5] && h[6] <= 64 && h[7] <= 3072) {
        const uint32_t st = (h[7] + h[6] + 16 + 15) & ~15u;
        if ((uint64_t)st * n <= (1ull << 31)) leaf_stride = st;
    }

    // ---- top-down: one launch per BFS level, or the whole BFS in one single-CTA launch for small tries ----
    std::vector<uint32_t> level_beg, level_cnt, level_ext;
    uint32_t beg = 0, cnt = h[0];
    if (cnt && leaf_stride && n <= 8192) {
        bfs_small_kernel<<<1, 1024, 0, s>>>(k, t, cnt, MAXL, bfs_levels);
        ctx->stats.launches++;
        std::vector<uint32_t> hl(2 + 3 * MAXL);
        CU(cudaMemcpyAsync(hl.data(), bfs_levels, 4 * hl.size(), cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        if (hl[1 + 3 * MAXL] != 0) return PHANT_GPU_E_INVALID;
        for (uint32_t l = 0; l < hl[0]; ++l) { level_beg.push_back(hl[1 + 3 * l]); level_cnt.push_back(hl[2 + 3 * l]); level_ext.push_back(hl[3 + 3 * l]); }
        cnt = 0;
    }
    while (cnt) {
        CU(cudaMemsetAsync(counters + 1, 0, 8, s));
        expand_kernel<<<grid1d(device, cnt, 128, 16), 128, 0, s>>>(k, t, beg, cnt, beg + cnt, counters);
        ctx->stats.launches++;
        CU(cudaMemcpyAsync(h, counters, 32, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        level_beg.push_back(beg); level_cnt.push_back(cnt); level_ext.push_back(h[2]);
        beg += cnt;
        cnt = h[1];
        if ((uint64_t)beg + cnt > cap) return PHANT_GPU_E_CUDA; // cannot happen: a trie over n keys has < n branch units
    }

    // Two arena layouts.  General: exact sizes, exclusive scan, one read-back of the total per pass.  Slots (leaf_stride != 0:
    // the caller vouches that no key is a prefix of another -- so no branch carries a value -- and bounds the leaf size):
    // every node gets a fixed-stride slot, the Keccak kernel takes (offset, length) pairs, and no pass needs a scan or
    // a host round trip.  Small tries are launch-bound, so this halves their latency.
    const bool slots = leaf_stride != 0;
    constexpr uint32_t BRANCH_STRIDE = 544, EXT_STRIDE = 128;
    uint32_t max_level = 1;
    for (uint32_t c : level_cnt) if (c > max_level) max_level = c;
    // what the largest level sizes: one unit pass's sizes, the branch and extension offsets, and the digests
    uint64_t *unit_size, *branch_off, *ext_off;
    uint8_t* unit_digests;
    RC(carve(ctx, ctx->fo_level, [&](Carve& c) {
        unit_size = c.take<uint64_t>(max_level + 2); branch_off = c.take<uint64_t>(max_level + 2); ext_off = c.take<uint64_t>(max_level + 2);
        unit_digests = c.take<uint8_t>(32ull * max_level);
    }));
    if (slots) {
        fixed_offsets_kernel<<<grid1d(device, n + 1, 256), 256, 0, s>>>(leaf_off, n, leaf_stride);
        fixed_offsets_kernel<<<grid1d(device, max_level + 1, 256), 256, 0, s>>>(branch_off, max_level, BRANCH_STRIDE);
        fixed_offsets_kernel<<<grid1d(device, max_level + 1, 256), 256, 0, s>>>(ext_off, max_level, EXT_STRIDE);
        ctx->stats.launches += 3;
    }

    // One pass over cnt nodes of one kind (forest_export_kernel's `what`: 0 leaves, 1 one level's branch units beg.., 2 its
    // extensions): sizes, offsets and one read-back of the total (general layout; slots: offs holds the fixed offsets), the
    // RLP into the kind's arena, the hash, the references and, when exporting, the nodes on a proof path.  size(sizes) and
    // encode(offs, arena, size_out) launch the kind's two kernels.
    auto pass = [&](uint32_t what, uint32_t cnt, const uint32_t* ids, uint32_t beg, auto&& size, auto&& encode) -> int {
        uint64_t* sizes = what ? unit_size : leaf_size;
        uint64_t* offs = what == 0 ? leaf_off : what == 1 ? branch_off : ext_off;
        uint8_t* digests = what ? unit_digests : ids ? leaf_compact_digests : leaf_digests;
        DevBuf& rlp = what ? ctx->fo_unit_rlp : ctx->fo_leaf_rlp;
        if (!slots) size(sizes);
        uint64_t total = (uint64_t)cnt * (what == 0 ? leaf_stride : what == 1 ? BRANCH_STRIDE : EXT_STRIDE);
        if (!slots) {
            RC(scan_sizes(ctx, sizes, offs, cnt));
            CU(cudaMemcpyAsync(&total, offs + cnt, 8, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
        }
        RC(rlp.reserve(ctx, total + 64));
        const uint8_t* arena = (const uint8_t*)rlp.ptr;
        const uint64_t* lens = slots ? sizes : nullptr;
        encode(offs, (uint8_t*)rlp.ptr, slots ? sizes : nullptr);
        ctx->stats.launches += slots ? 1 : 2;
        if (slots) RC(ctx->hash_slots(arena, offs, sizes, cnt, digests));
        else RC(ctx->hash_csr(arena, offs, cnt, total, digests));
        finalize_ref_kernel<<<grid1d(device, cnt, 256), 256, 0, s>>>(cnt, ids, beg, offs, lens, arena, digests, what ? n : 0, t,
                                                                     what ? t.top_digest : ids ? leaf_digests : nullptr);
        ctx->stats.launches++;
        if (f.xp) {
            forest_export_kernel<<<grid1d(device, cnt, 256), 256, 0, s>>>(k, t, *f.xp, what, cnt, ids, beg, offs, lens, arena, digests);
            ctx->stats.launches++;
        }
        return PHANT_GPU_OK;
    };

    trf.mark("    forest: check + BFS");
    // ---- leaves (only those the cache cannot answer) ----
    if (n) {
        uint32_t m = n;                 // leaves to encode
        const uint32_t* ids = nullptr;  // their key indices (nullptr = all, in order)
        if (f.leaf_cache) {
            leaf_cache_probe_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(t, n, f.leaf_cache, leaf_digests, cache_flag);
            CU(cudaMemsetAsync(cache_flag + n, 0, 4, s));
            RC(scan_u32(ctx, cache_flag, cache_pos, n + 1));
            compact_iota_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(cache_flag, cache_pos, n, cache_list);
            CU(cudaMemcpyAsync(&m, cache_pos + n, 4, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            ids = cache_list;
            ctx->stats.launches += 3;
        }
        if (m)
            RC(pass(0, m, ids, 0, [&](uint64_t* sizes) { leaf_size_kernel<<<grid1d(device, m, 256), 256, 0, s>>>(k, vals, t, m, sizes, ids); },
                    [&](const uint64_t* offs, uint8_t* arena, uint64_t* size_out) {
                        leaf_encode_kernel<<<grid1d(device, m, 256, 32), 256, 0, s>>>(k, vals, t, m, offs, arena, size_out, ids);
                    }));
        if (f.leaf_cache_out) {
            leaf_cache_store_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(t, n, leaf_digests, f.leaf_cache_out);
            ctx->stats.launches++;
        }
    }

    trf.mark("    forest: leaves");
    // ---- units, deepest level first: branch, then the extension above it where there is one ----
    for (int L = (int)level_beg.size() - 1; L >= 0; --L) {
        const uint32_t lb = level_beg[L], lc = level_cnt[L], le = level_ext[L];
        RC(pass(1, lc, nullptr, lb, [&](uint64_t* sizes) { branch_size_kernel<<<grid1d(device, lc, 128), 128, 0, s>>>(k, vals, t, n, lb, lc, sizes); },
                [&](const uint64_t* offs, uint8_t* arena, uint64_t* size_out) {
                    branch_encode_kernel<<<grid1d(device, lc, 256, 32), 256, 0, s>>>(k, vals, t, n, lb, lc, offs, size_out, slots, arena);
                }));
        if (le) {
            const uint32_t* ids = t.ext_list + lb;
            RC(pass(2, le, ids, 0, [&](uint64_t* sizes) { ext_size_kernel<<<grid1d(device, le, 128), 128, 0, s>>>(k, t, n, ids, le, sizes); },
                    [&](const uint64_t* offs, uint8_t* arena, uint64_t* size_out) {
                        ext_encode_kernel<<<grid1d(device, le, 128), 128, 0, s>>>(k, t, n, ids, le, offs, arena, size_out);
                    }));
        }
    }
    trf.mark("    forest: units bottom-up");
    gather_roots_kernel<<<grid1d(device, n_seg, 128), 128, 0, s>>>(t, n_seg, leaf_digests, f.roots);
    ctx->stats.launches++;
    CU(cudaGetLastError());
    return PHANT_GPU_OK;
}

} // namespace

// ------------------------------------------------------------------------------------------------
// M
// ------------------------------------------------------------------------------------------------
extern "C" int phant_gpu_mpt_root(phant_gpu_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* vals,
                                  const uint64_t* val_off, uint64_t n, uint8_t out_root[32])
{
    if (!ctx || !out_root || (n && (!key_off || !val_off))) return PHANT_GPU_E_INVALID;
    if (n >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    if (n == 0) { memcpy(out_root, EMPTY_ROOT_H, 32); return PHANT_GPU_OK; }
    cudaStream_t s = ctx->stream;
    const uint8_t* d_keys = keys; const uint32_t* d_koff = key_off; const uint8_t* d_vals = vals; const uint64_t* d_voff = val_off;
    if (!(ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS)) {
        for (uint64_t i = 0; i < n; ++i)
            if (key_off[i + 1] < key_off[i] || val_off[i + 1] < val_off[i]) return PHANT_GPU_E_INVALID;
        const uint64_t kb = key_off[n], vb = val_off[n];
        if ((kb && !keys) || (vb && !vals)) return PHANT_GPU_E_INVALID;
        uint8_t *dk, *dv;
        uint64_t* dvo;
        uint32_t* dko;
        RC(carve(ctx, ctx->d_msgs, [&](Carve& c) { dk = c.take<uint8_t>(kb); dv = c.take<uint8_t>(vb); }));
        RC(carve(ctx, ctx->d_off, [&](Carve& c) { dvo = c.take<uint64_t>(n + 1); dko = c.take<uint32_t>(n + 1); }));
        if (kb) CU(cudaMemcpyAsync(dk, keys, kb, cudaMemcpyHostToDevice, s));
        if (vb) CU(cudaMemcpyAsync(dv, vals, vb, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dko, key_off, 4 * (n + 1), cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dvo, val_off, 8 * (n + 1), cudaMemcpyHostToDevice, s));
        ctx->stats.h2d_bytes += kb + vb + 12 * (n + 1);
        d_keys = dk; d_koff = dko; d_vals = dv; d_voff = dvo;
    }
    RC(ctx->d_first.reserve(ctx, 64));
    uint32_t seg[2] = {0, (uint32_t)n};
    CU(cudaMemcpyAsync(ctx->d_first.ptr, seg, 8, cudaMemcpyHostToDevice, s));
    RC(ctx->d_roots.reserve(ctx, 32));
    RC(build_forest(ctx, {.keys = d_keys, .key_off = d_koff, .vals = d_vals, .val_off = d_voff, .n = (uint32_t)n,
                          .seg_off = (const uint32_t*)ctx->d_first.ptr, .n_seg = 1, .roots = (uint8_t*)ctx->d_roots.ptr}));
    RC(copy_out(ctx, out_root, ctx->d_roots.ptr, 32));
    CU(cudaStreamSynchronize(s));
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_mpt_roots(phant_gpu_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* vals,
                                   const uint64_t* val_off, const uint32_t* seg_off, uint64_t n_tries, uint8_t* out_roots)
{
    if (!ctx || (n_tries && (!seg_off || !out_roots))) return PHANT_GPU_E_INVALID;
    if (n_tries == 0) return PHANT_GPU_OK;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // the batched form takes host arrays
    if (n_tries >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    for (uint64_t t = 0; t < n_tries; ++t) if (seg_off[t + 1] < seg_off[t]) return PHANT_GPU_E_INVALID;
    if (seg_off[0] != 0) return PHANT_GPU_E_INVALID;
    const uint64_t n = seg_off[n_tries];
    if (n >= (1ull << 30) || (n && (!key_off || !val_off))) return PHANT_GPU_E_INVALID;
    for (uint64_t i = 0; i < n; ++i)
        if (key_off[i + 1] < key_off[i] || val_off[i + 1] < val_off[i]) return PHANT_GPU_E_INVALID;
    const uint64_t kb = n ? key_off[n] : 0, vb = n ? val_off[n] : 0;
    if ((kb && !keys) || (vb && !vals)) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    // segment id of every key (the sortedness check must not compare across tries)
    std::vector<uint32_t> seg_of_key(n ? n : 1);
    for (uint64_t t = 0; t < n_tries; ++t)
        for (uint32_t i = seg_off[t]; i < seg_off[t + 1]; ++i) seg_of_key[i] = (uint32_t)t;
    uint8_t *dk, *dv;
    uint64_t* dvo;
    uint32_t *dko, *dseg, *dsok;
    RC(carve(ctx, ctx->d_msgs, [&](Carve& c) { dk = c.take<uint8_t>(kb); dv = c.take<uint8_t>(vb); }));
    RC(carve(ctx, ctx->d_off, [&](Carve& c) { dvo = c.take<uint64_t>(n + 1); dko = c.take<uint32_t>(n + 1); }));
    RC(carve(ctx, ctx->d_first, [&](Carve& c) { dseg = c.take<uint32_t>(n_tries + 1); dsok = c.take<uint32_t>(n + 1); }));
    RC(ctx->d_roots.reserve(ctx, 32 * n_tries));
    static const uint32_t zero_off[2] = {0, 0};
    static const uint64_t zero_off64[2] = {0, 0};
    if (kb) CU(cudaMemcpyAsync(dk, keys, kb, cudaMemcpyHostToDevice, s));
    if (vb) CU(cudaMemcpyAsync(dv, vals, vb, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dko, n ? key_off : zero_off, 4 * (n + 1), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dvo, n ? val_off : zero_off64, 8 * (n + 1), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dseg, seg_off, 4 * (n_tries + 1), cudaMemcpyHostToDevice, s));
    if (n) CU(cudaMemcpyAsync(dsok, seg_of_key.data(), 4 * n, cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s)); // seg_of_key is a local vector: the copy must finish before it goes out of scope
    ctx->stats.h2d_bytes += kb + vb + 16 * (n + 1) + 4 * (n_tries + 1);
    RC(build_forest(ctx, {.keys = dk, .key_off = dko, .vals = dv, .val_off = dvo, .n = (uint32_t)n, .seg_off = dseg, .n_seg = (uint32_t)n_tries,
                          .seg_of_key = dsok, .roots = (uint8_t*)ctx->d_roots.ptr}));
    RC(copy_out(ctx, out_roots, ctx->d_roots.ptr, 32 * n_tries));
    CU(cudaStreamSynchronize(s));
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// S: state root
// ------------------------------------------------------------------------------------------------
namespace {

// non-zero slots -> (segment = account, hashed key index); also the rlp(trim(value)) size
__global__ void slot_flag_kernel(const uint8_t* __restrict__ vals32, uint64_t n_slots, uint8_t* __restrict__ keep)
{
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* p = reinterpret_cast<const uint4*>(vals32 + 32 * i);
        const uint4 a = p[0], b = p[1];
        keep[i] = (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) ? 1 : 0;
    }
}
__global__ void slot_account_kernel(const uint64_t* __restrict__ slot_off, uint32_t n_acc, uint32_t* __restrict__ acc_of_slot)
{
    // one warp per account, lanes stride over its slots
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a < n_acc; a += (gridDim.x * blockDim.x) >> 5)
        for (uint64_t s = slot_off[a] + lane; s < slot_off[a + 1]; s += 32) acc_of_slot[s] = a;
}
// key word w (0 = most significant 8 bytes, big endian) of the 32-byte hashes, for the LSD radix passes
__global__ void key_word_kernel(const uint8_t* __restrict__ hashes, const uint32_t* __restrict__ perm, uint32_t n, uint32_t w,
                                uint64_t* __restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint8_t* h = hashes + 32ull * perm[i] + 8 * w;
        uint64_t v = 0;
        for (int b = 0; b < 8; ++b) v = (v << 8) | h[b];
        out[i] = v;
    }
}
__global__ void gather_u32_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ perm, uint32_t n, uint32_t* __restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = src[perm[i]];
}
__global__ void iota_kernel(uint32_t* p, uint32_t n)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = i;
}
__global__ void storage_value_size_kernel(const uint8_t* __restrict__ vals32, const uint32_t* __restrict__ slot_of_sorted, uint32_t n,
                                          uint64_t* __restrict__ size)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint8_t* v = vals32 + 32ull * slot_of_sorted[i];
        uint32_t z = 0;
        while (z < 32 && v[z] == 0) ++z;
        const uint32_t len = 32 - z;
        size[i] = (len == 1 && v[z] < 0x80) ? 1 : 1 + len;
    }
}
__global__ void storage_fill_kernel(const uint8_t* __restrict__ slot_hash, const uint8_t* __restrict__ vals32,
                                    const uint32_t* __restrict__ slot_of_sorted, uint32_t n, const uint64_t* __restrict__ val_off,
                                    uint8_t* __restrict__ keys_out, uint32_t* __restrict__ key_off, uint8_t* __restrict__ vals_out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) {
        key_off[i] = 32u * i;
        if (i == n) break;
        const uint32_t sl = slot_of_sorted[i];
        for (int b = 0; b < 32; ++b) keys_out[32ull * i + b] = slot_hash[32ull * sl + b];
        const uint8_t* v = vals32 + 32ull * sl;
        uint32_t z = 0;
        while (z < 32 && v[z] == 0) ++z;
        const uint32_t len = 32 - z;
        uint8_t* o = vals_out + val_off[i];
        if (!(len == 1 && v[z] < 0x80)) *o++ = (uint8_t)(0x80 + len);
        for (uint32_t b = 0; b < len; ++b) o[b] = v[z + b];
    }
}
// segment offsets of the sorted, compacted slots: seg_off[a] = first sorted slot of account a (counts then scan)
__global__ void count_per_account_kernel(const uint32_t* __restrict__ acc_sorted, uint32_t n, uint32_t* __restrict__ counts)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) atomicAdd(&counts[acc_sorted[i]], 1u);
}
// account leaf value rlp([nonce, balance, storage_root, code_hash]) in sorted account order
__global__ void account_size_kernel(const uint64_t* __restrict__ nonce, const uint8_t* __restrict__ balance32,
                                    const uint32_t* __restrict__ acc_of_sorted, uint32_t n, uint64_t* __restrict__ size)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t a = acc_of_sorted[i];
        const uint64_t nn = nonce[a];
        const uint32_t nl = be_len(nn);
        uint64_t payload = (nl == 0) ? 1 : ((nl == 1 && nn < 0x80) ? 1 : 1 + nl);
        const uint8_t* b = balance32 + 32ull * a;
        uint32_t z = 0;
        while (z < 32 && b[z] == 0) ++z;
        const uint32_t bl = 32 - z;
        payload += (bl == 0) ? 1 : ((bl == 1 && b[z] < 0x80) ? 1 : 1 + bl);
        payload += 33 + 33;
        size[i] = hdr_size(payload) + payload;
    }
}
__global__ void account_fill_kernel(const uint64_t* __restrict__ nonce, const uint8_t* __restrict__ balance32,
                                    const uint8_t* __restrict__ storage_roots, const uint8_t* __restrict__ code_hashes,
                                    const uint8_t* __restrict__ addr_hashes, const uint32_t* __restrict__ acc_of_sorted, uint32_t n,
                                    const uint64_t* __restrict__ val_off, uint8_t* __restrict__ keys_out, uint32_t* __restrict__ key_off,
                                    uint8_t* __restrict__ vals_out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) {
        key_off[i] = 32u * i;
        if (i == n) break;
        const uint32_t a = acc_of_sorted[i];
        for (int b = 0; b < 32; ++b) keys_out[32ull * i + b] = addr_hashes[32ull * a + b];
        uint8_t* out = vals_out + val_off[i];
        const uint64_t total = val_off[i + 1] - val_off[i];
        uint32_t hdr = 1;
        for (uint32_t cand = 1; cand <= 3; ++cand)
            if (hdr_size(total - cand) == cand) { hdr = cand; break; }
        uint8_t* q = out + put_hdr(out, total - hdr, 0xc0, 0xf7);
        const uint64_t nn = nonce[a];
        const uint32_t nl = be_len(nn);
        if (nl == 0) *q++ = 0x80;
        else if (nl == 1 && nn < 0x80) *q++ = (uint8_t)nn;
        else { *q++ = (uint8_t)(0x80 + nl); for (uint32_t b = 0; b < nl; ++b) *q++ = (uint8_t)(nn >> (8 * (nl - 1 - b))); }
        const uint8_t* bal = balance32 + 32ull * a;
        uint32_t z = 0;
        while (z < 32 && bal[z] == 0) ++z;
        const uint32_t bl = 32 - z;
        if (bl == 0) *q++ = 0x80;
        else if (bl == 1 && bal[z] < 0x80) *q++ = bal[z];
        else { *q++ = (uint8_t)(0x80 + bl); for (uint32_t b = 0; b < bl; ++b) *q++ = bal[z + b]; }
        *q++ = 0xa0;
        for (int b = 0; b < 32; ++b) *q++ = storage_roots[32ull * a + b];
        *q++ = 0xa0;
        for (int b = 0; b < 32; ++b) *q++ = code_hashes[32ull * a + b];
    }
}
__global__ void gather_rows32_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t cnt, uint8_t* __restrict__ dst)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
        const uint4* p = reinterpret_cast<const uint4*>(src + 32ull * idx[i]);
        uint4* q = reinterpret_cast<uint4*>(dst + 32ull * i);
        q[0] = p[0];
        q[1] = p[1];
    }
}

// stable LSD radix sort of n items by (segment, 32-byte big-endian hash): perm_out[i] = index of the i-th smallest
int sort_by_segment_and_hash(phant_gpu_ctx* ctx, const uint8_t* d_hashes, const uint32_t* d_seg /*nullable*/, uint32_t n, uint32_t* d_perm_out,
                             DevBuf& scratch)
{
    cudaStream_t s = ctx->stream;
    const int device = ctx->device;
    if (n == 0) return PHANT_GPU_OK;
    uint64_t *kin, *kout;
    uint32_t *pa, *pb, *sk;
    RC(carve(ctx, scratch, [&](Carve& c) {
        kin = c.take<uint64_t>(n); kout = c.take<uint64_t>(n); pa = c.take<uint32_t>(n); pb = c.take<uint32_t>(n); sk = c.take<uint32_t>(n);
    }));
    iota_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(pa, n);
    uint32_t* cur = pa;
    uint32_t* nxt = pb;
    for (int w = 3; w >= 0; --w) { // least significant word first
        key_word_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(d_hashes, cur, n, (uint32_t)w, kin);
        RC(cub_call(ctx, [&](void* tmp, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(tmp, b, (const uint64_t*)kin, kout, (const uint32_t*)cur, nxt, (int64_t)n, 0, 64, s);
        }));
        uint32_t* tsw = cur; cur = nxt; nxt = tsw;
        ctx->stats.launches += 2;
    }
    if (d_seg) {
        gather_u32_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(d_seg, cur, n, sk);
        RC(cub_call(ctx, [&](void* tmp, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(tmp, b, (const uint32_t*)sk, (uint32_t*)kout, (const uint32_t*)cur, nxt, (int64_t)n, 0, 32, s);
        }));
        uint32_t* tsw = cur; cur = nxt; nxt = tsw;
        ctx->stats.launches += 2;
    }
    CU(cudaMemcpyAsync(d_perm_out, cur, 4ull * n, cudaMemcpyDeviceToDevice, s));
    return PHANT_GPU_OK;
}

// seg_off[v] = first sorted key whose top nibble is >= v (v = 0..16): the 16 subtrees under the root branch
__global__ void top_nibble_segments_kernel(const uint8_t* __restrict__ sorted_keys32, uint32_t n, uint32_t* __restrict__ seg_off)
{
    const uint32_t v = threadIdx.x;
    if (v > 16) return;
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if ((uint32_t)(sorted_keys32[32ull * mid] >> 4) < v) a = mid + 1; else b = mid;
    }
    seg_off[v] = a;
}
} // namespace

// S and its sharded form.  subtree_mask == nullptr: out = the state root (32 bytes).  Otherwise: out = 16 x 32 bytes, the
// hashes of the subtrees under the root branch's 16 slots (accounts grouped by the top nibble of keccak(addr), tries built
// from nibble 1 on), *subtree_mask bit v = slot v is populated.  An account leaf is >= 70 bytes, so a populated slot's
// reference is always the 32-byte hash.
static int state_root_impl(phant_gpu_ctx* ctx, const phant_gpu_accounts* a, uint8_t* out_root, uint32_t* subtree_mask)
{
    if (!ctx || !a || !out_root) return PHANT_GPU_E_INVALID;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // S takes host tables (it is the StateDB flattening)
    const uint64_t n = a->n_accounts;
    if (n == 0) {
        if (subtree_mask) { *subtree_mask = 0; memset(out_root, 0, 16 * 32); }
        else memcpy(out_root, EMPTY_ROOT_H, 32);
        return PHANT_GPU_OK;
    }
    if (n >= (1ull << 30) || !a->addr20 || !a->nonce || !a->balance32 || !a->code_off || !a->slot_off) return PHANT_GPU_E_INVALID;
    for (uint64_t i = 0; i < n; ++i)
        if (a->code_off[i + 1] < a->code_off[i] || a->slot_off[i + 1] < a->slot_off[i]) return PHANT_GPU_E_INVALID;
    const uint64_t code_bytes = a->code_off[n] - a->code_off[0], n_slots = a->slot_off[n] - a->slot_off[0];
    if (a->code_off[0] != 0 || a->slot_off[0] != 0) return PHANT_GPU_E_INVALID;
    if ((code_bytes && !a->code) || (n_slots && (!a->slot_keys32 || !a->slot_vals32)) || n_slots >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;

    // ---- stage the tables (one arena in st_in) ----
    uint8_t *addr, *bal, *code, *skey, *sval;
    uint64_t *nonce, *code_off, *slot_off;
    RC(carve(ctx, ctx->st_in, [&](Carve& c) {
        addr = c.take<uint8_t>(20 * n); nonce = c.take<uint64_t>(n); bal = c.take<uint8_t>(32 * n);
        code = c.take<uint8_t>(code_bytes + 64); code_off = c.take<uint64_t>(n + 1);
        skey = c.take<uint8_t>(32 * n_slots + 64); sval = c.take<uint8_t>(32 * n_slots + 64); slot_off = c.take<uint64_t>(n + 1);
    }));
    CU(cudaMemcpyAsync(addr, a->addr20, 20 * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(nonce, a->nonce, 8 * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(bal, a->balance32, 32 * n, cudaMemcpyHostToDevice, s));
    if (code_bytes) CU(cudaMemcpyAsync(code, a->code, code_bytes, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(code_off, a->code_off, 8 * (n + 1), cudaMemcpyHostToDevice, s));
    if (n_slots) {
        CU(cudaMemcpyAsync(skey, a->slot_keys32, 32 * n_slots, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(sval, a->slot_vals32, 32 * n_slots, cudaMemcpyHostToDevice, s));
    }
    CU(cudaMemcpyAsync(slot_off, a->slot_off, 8 * (n + 1), cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += 60 * n + code_bytes + 64 * n_slots + 16 * (n + 1);

    // ---- hashes: keccak(addr), keccak(code), keccak(slot key) (batched Keccak kernel, three launches) ----
    uint8_t *h_addr, *h_code, *h_slot, *sroots;
    uint64_t* fixed;
    RC(carve(ctx, ctx->st_hash, [&](Carve& c) {
        h_addr = c.take<uint8_t>(32 * n); h_code = c.take<uint8_t>(32 * n); h_slot = c.take<uint8_t>(32 * n_slots + 32);
        sroots = c.take<uint8_t>(32 * n); fixed = c.take<uint64_t>((n > n_slots ? n : n_slots) + 1);
    }));
    fixed_offsets_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(fixed, n, 20);
    ctx->stats.launches++;
    RC(ctx->hash_csr(addr, fixed, n, 20 * n, h_addr));
    RC(ctx->hash_csr(code, code_off, n, code_bytes, h_code));
    if (n_slots) {
        fixed_offsets_kernel<<<grid1d(dev, n_slots, 256), 256, 0, s>>>(fixed, n_slots, 32);
        ctx->stats.launches++;
        RC(ctx->hash_csr(skey, fixed, n_slots, 32 * n_slots, h_slot));
    }

    // ---- storage tries: drop zero slots, sort by (account, hashed key), build all tries as one forest ----
    uint32_t *seg_cnt, *seg_off, *acc_of_slot, *kept, *n_kept, *perm, *slot_sorted;
    uint8_t* keep;
    RC(carve(ctx, ctx->st_seg, [&](Carve& c) {
        seg_cnt = c.take<uint32_t>(n + 2); seg_off = c.take<uint32_t>(n + 2); acc_of_slot = c.take<uint32_t>(n_slots + 1);
        kept = c.take<uint32_t>(n_slots + 1);        // compacted -> slot
        n_kept = c.take<uint32_t>(1);
        perm = c.take<uint32_t>(n_slots + 1);        // sorted -> compacted
        slot_sorted = c.take<uint32_t>(n_slots + 1); // sorted -> slot
        keep = c.take<uint8_t>(n_slots + 1);
    }));
    uint32_t m = 0; // kept slots
    if (n_slots) {
        slot_flag_kernel<<<grid1d(dev, n_slots, 256), 256, 0, s>>>(sval, n_slots, keep);
        slot_account_kernel<<<grid1d(dev, n, 256, 32), 256, 0, s>>>(slot_off, (uint32_t)n, acc_of_slot);
        iota_kernel<<<grid1d(dev, n_slots, 256), 256, 0, s>>>(perm, (uint32_t)n_slots);
        ctx->stats.launches += 3;
        RC(cub_call(ctx, [&](void* tmp, size_t& b) {
            return cub::DeviceSelect::Flagged(tmp, b, (const uint32_t*)perm, (const uint8_t*)keep, kept, n_kept, (int64_t)n_slots, s);
        }));
        CU(cudaMemcpyAsync(&m, n_kept, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    CU(cudaMemsetAsync(seg_cnt, 0, 4ull * (n + 2), s));
    if (m) {
        // gather the kept slots' hashes / accounts into compact arrays, sort, and lay the forest inputs out
        uint8_t *ch, *fk, *fv;
        uint32_t *cacc, *acc_sorted, *fko;
        uint64_t *fvs, *fvo;
        RC(carve(ctx, ctx->st_tmp, [&](Carve& c) {
            ch = c.take<uint8_t>(32ull * m);   // compact hashes
            cacc = c.take<uint32_t>(m);        // compact account ids
            acc_sorted = c.take<uint32_t>(m);
            fk = c.take<uint8_t>(32ull * m);   // forest keys
            fko = c.take<uint32_t>(m + 1); fvs = c.take<uint64_t>(m + 1); fvo = c.take<uint64_t>(m + 1); fv = c.take<uint8_t>(33ull * m);
        }));
        gather_rows32_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(h_slot, kept, m, ch);
        gather_u32_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(acc_of_slot, kept, m, cacc);
        ctx->stats.launches += 2;
        RC(sort_by_segment_and_hash(ctx, ch, cacc, m, perm, ctx->st_sort));
        gather_u32_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(kept, perm, m, slot_sorted);
        gather_u32_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(cacc, perm, m, acc_sorted);
        count_per_account_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(acc_sorted, m, seg_cnt);
        storage_value_size_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(sval, slot_sorted, m, fvs);
        ctx->stats.launches += 4;
        RC(scan_sizes(ctx, fvs, fvo, m));
        storage_fill_kernel<<<grid1d(dev, m + 1, 256), 256, 0, s>>>(h_slot, sval, slot_sorted, m, fvo, fk, fko, fv);
        ctx->stats.launches++;
        RC(scan_u32(ctx, seg_cnt, seg_off, n + 1));
        RC(build_forest(ctx, {.keys = fk, .key_off = fko, .vals = fv, .val_off = fvo, .n = m, .seg_off = seg_off, .n_seg = (uint32_t)n,
                              .seg_of_key = acc_sorted, .roots = sroots, .slot_stride = /*32-byte keys, values <= 33 B*/ 96}));
    } else {
        CU(cudaMemsetAsync(seg_off, 0, 4ull * (n + 2), s));
        RC(build_forest(ctx, {.seg_off = seg_off, .n_seg = (uint32_t)n, .roots = sroots})); // every storage trie empty
    }

    // ---- account trie ----
    uint32_t *acc_perm, *ako;
    uint8_t *ak, *av;
    uint64_t *avs, *avo;
    RC(carve(ctx, ctx->st_acc, [&](Carve& c) {
        acc_perm = c.take<uint32_t>(n); ak = c.take<uint8_t>(32ull * n); ako = c.take<uint32_t>(n + 1);
        avs = c.take<uint64_t>(n + 1); avo = c.take<uint64_t>(n + 1); av = c.take<uint8_t>(112ull * n);
    }));
    RC(sort_by_segment_and_hash(ctx, h_addr, nullptr, (uint32_t)n, acc_perm, ctx->st_sort));
    account_size_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(nonce, bal, acc_perm, (uint32_t)n, avs);
    ctx->stats.launches++;
    RC(scan_sizes(ctx, avs, avo, n));
    account_fill_kernel<<<grid1d(dev, n + 1, 256), 256, 0, s>>>(nonce, bal, sroots, h_code, h_addr, acc_perm, (uint32_t)n, avo, ak, ako, av);
    ctx->stats.launches++;
    RC(ctx->d_first.reserve(ctx, 128));
    RC(ctx->d_roots.reserve(ctx, 16 * 32));
    if (subtree_mask) {
        uint32_t seg[17];
        top_nibble_segments_kernel<<<1, 32, 0, s>>>(ak, (uint32_t)n, (uint32_t*)ctx->d_first.ptr);
        ctx->stats.launches++;
        RC(copy_out(ctx, seg, ctx->d_first.ptr, sizeof seg));
        RC(build_forest(ctx, {.keys = ak, .key_off = ako, .vals = av, .val_off = avo, .n = (uint32_t)n, .seg_off = (const uint32_t*)ctx->d_first.ptr,
                              .n_seg = 16, .roots = (uint8_t*)ctx->d_roots.ptr, .slot_stride = 160, .start_depth = /*the root branch consumed nibble 0*/ 1}));
        RC(copy_out(ctx, out_root, ctx->d_roots.ptr, 16 * 32));
        CU(cudaStreamSynchronize(s));
        uint32_t mask = 0;
        for (int v = 0; v < 16; ++v) {
            if (seg[v + 1] > seg[v]) mask |= 1u << v;
            else memset(out_root + 32 * v, 0, 32);
        }
        *subtree_mask = mask;
        return PHANT_GPU_OK;
    }
    uint32_t seg[2] = {0, (uint32_t)n};
    CU(cudaMemcpyAsync(ctx->d_first.ptr, seg, 8, cudaMemcpyHostToDevice, s));
    RC(build_forest(ctx, {.keys = ak, .key_off = ako, .vals = av, .val_off = avo, .n = (uint32_t)n, .seg_off = (const uint32_t*)ctx->d_first.ptr,
                          .n_seg = 1, .roots = (uint8_t*)ctx->d_roots.ptr, .slot_stride = /*32-byte keys, account RLP <= 110 B*/ 160}));
    RC(copy_out(ctx, out_root, ctx->d_roots.ptr, 32));
    CU(cudaStreamSynchronize(s));
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_state_root(phant_gpu_ctx* ctx, const phant_gpu_accounts* a, uint8_t out_root[32])
{
    return state_root_impl(ctx, a, out_root, nullptr);
}

extern "C" int phant_gpu_state_subtree_roots(phant_gpu_ctx* ctx, const phant_gpu_accounts* a, uint8_t out_roots[16 * 32], uint32_t* out_mask)
{
    if (!out_mask) return PHANT_GPU_E_INVALID;
    return state_root_impl(ctx, a, out_roots, out_mask);
}

// ------------------------------------------------------------------------------------------------
// U: resident complete trie
// ------------------------------------------------------------------------------------------------
struct SparseTrie;
struct phant_gpu_trie {
    phant_gpu_ctx* ctx;
    uint32_t kind = 0;
    uint32_t depth;
    std::vector<uint8_t*> level; // kind 0: level[l] = 16^l hashes
    DevBuf store;
    DevBuf work, leaf_rlp;       // kind 0's scratch: counter words and the update's position lists; the general leaf path's RLP
    SparseTrie* sp = nullptr;    // kind 1
};

namespace {

__device__ __forceinline__ uint64_t sm64(uint64_t& s)
{
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__global__ void ctrie_fill_leaves_kernel(uint64_t seed, uint64_t n_leaves, uint8_t* __restrict__ out)
{
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_leaves; j += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t s = seed ^ (0xC4ull * 0xA24BAED4963EE407ull) ^ (j * 0xD1342543DE82EF95ull);
        (void)sm64(s);
        uint64_t* o = reinterpret_cast<uint64_t*>(out + 32 * j);
        for (int w = 0; w < 4; ++w) o[w] = sm64(s); // little-endian bytes == the oracle's byte order
    }
}
__global__ void ctrie_scatter_kernel(const uint8_t* __restrict__ digests, const uint32_t* __restrict__ pos, uint64_t cnt, uint8_t* __restrict__ level)
{
    for (uint64_t u = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; u < cnt; u += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* p = reinterpret_cast<const uint4*>(digests + 32 * u);
        uint4* q = reinterpret_cast<uint4*>(level + 32ull * (pos ? pos[u] : u));
        q[0] = p[0];
        q[1] = p[1];
    }
}
// dirty leaves: position = first `depth` nibbles of the key; leaf RLP = list[hp(nibbles[depth..64), leaf), value]
__global__ void ctrie_leaf_pos_kernel(const uint8_t* __restrict__ keys32, uint64_t n, uint32_t depth, uint32_t* __restrict__ pos)
{
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t* key = keys32 + 32 * k;
        uint32_t p = 0;
        for (uint32_t i = 0; i < depth; ++i) p = p * 16 + ((i & 1) ? (key[i >> 1] & 15u) : (key[i >> 1] >> 4));
        pos[k] = p;
    }
}
__global__ void ctrie_leaf_size_kernel(const uint8_t* __restrict__ vals, const uint32_t* __restrict__ val_off, uint64_t n, uint32_t depth,
                                       uint64_t* __restrict__ size)
{
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t cnt = 64 - depth, hpn = 1 + cnt / 2;
        const uint64_t vl = val_off[k + 1] - val_off[k];
        // the first hex-prefix byte is 0x20 or 0x3n: a lone byte < 0x80 encodes as itself
        const uint64_t payload = (hpn == 1 ? 1 : 1 + hpn) + str_size(vl, vl ? vals[val_off[k]] : 0);
        size[k] = hdr_size(payload) + payload;
    }
}
__global__ void ctrie_leaf_encode_kernel(const uint8_t* __restrict__ keys32, const uint8_t* __restrict__ vals, const uint32_t* __restrict__ val_off,
                                         uint64_t n, uint32_t depth, const uint64_t* __restrict__ aoff, uint8_t* __restrict__ arena)
{
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t* key = keys32 + 32 * k;
        const uint32_t cnt = 64 - depth, hpn = 1 + cnt / 2;
        const uint64_t vl = val_off[k + 1] - val_off[k];
        const uint8_t* v = vals + val_off[k];
        const uint64_t s_hp = hpn == 1 ? 1 : 1 + hpn, s_v = str_size(vl, vl ? v[0] : 0);
        uint8_t* out = arena + aoff[k];
        uint8_t* q = out + put_hdr(out, s_hp + s_v, 0xc0, 0xf7);
        if (hpn > 1) *q++ = (uint8_t)(0x80 + hpn);
        uint32_t i = depth;
#define KN(j) (((j) & 1) ? (key[(j) >> 1] & 15u) : (key[(j) >> 1] >> 4))
        if (cnt & 1) { *q++ = (uint8_t)(0x30 | KN(i)); ++i; } else *q++ = 0x20;
        for (; i < 64; i += 2) *q++ = (uint8_t)((KN(i) << 4) | KN(i + 1));
#undef KN
        if (s_v > vl) q += put_hdr(q, vl, 0x80, 0xb7);
        for (uint64_t b = 0; b < vl; ++b) q[b] = v[b];
    }
}

// ---- fused frontier kernels: encode in shared memory, hash, store -- one launch per level, no arena, no host sync ----
constexpr int FR_SLOT = 560;  // same geometry as the staged Keccak kernel's slots (16 x 35)
constexpr int FR_WARPS = 4;
constexpr int FR_SMEM = FR_WARPS * 32 * FR_SLOT + 16;

__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts8(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }

// byte stream -> aligned 32-bit shared-memory words; FILL (bytes pending in acc) is a compile-time constant everywhere
template <int FILL>
__device__ __forceinline__ void push_word(uint32_t& sa, uint32_t& acc, uint32_t h)
{
    if constexpr (FILL == 0) { sts32(sa, h); sa += 4; }
    else { sts32(sa, acc | (h << (8 * FILL))); sa += 4; acc = h >> (32 - 8 * FILL); }
}
template <int S>
__device__ __forceinline__ void push_child(uint32_t& sa, uint32_t& acc, const uint4 a, const uint4 b)
{
    // before child S the stream holds 3 + 33*S bytes: FILL = (3 + S) % 4; the 0xa0 marker goes first
    constexpr int F0 = (3 + S) % 4;
    if constexpr (F0 == 3) { sts32(sa, acc | (0xa0u << 24)); sa += 4; acc = 0; }
    else acc |= 0xa0u << (8 * F0);
    constexpr int F = (F0 + 1) % 4;
    push_word<F>(sa, acc, a.x); push_word<F>(sa, acc, a.y); push_word<F>(sa, acc, a.z); push_word<F>(sa, acc, a.w);
    push_word<F>(sa, acc, b.x); push_word<F>(sa, acc, b.y); push_word<F>(sa, acc, b.z); push_word<F>(sa, acc, b.w);
}

// Re-hash the dirty branch nodes of one level: parent p = parents[i] (i < *count), children = child_level[16p .. 16p+16).
// Each thread writes the 532-byte encoding f9 0211 | 16 x (a0 hash) | 80 (mpt.zig:218-247) into its shared-memory slot as
// aligned words, absorbs it with the product sponge, and stores the digest at level[p].
__global__ void __launch_bounds__(FR_WARPS * 32)
frontier_branch_kernel(const uint8_t* __restrict__ child_level, const uint32_t* __restrict__ parents, const uint32_t* __restrict__ count_ptr,
                       uint32_t bound, uint8_t* __restrict__ level, const uint32_t* __restrict__ refuse)
{
    extern __shared__ __align__(16) uint8_t fr_smem[];
    const uint32_t slot = (uint32_t)__cvta_generic_to_shared(fr_smem) + threadIdx.x * FR_SLOT;
    if (*refuse) return; // duplicate leaf positions: the update is refused as a whole
    uint32_t count = *count_ptr;
    if (count > bound) count = bound;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const uint32_t p = parents[i];
        const uint4* ch = reinterpret_cast<const uint4*>(child_level + 512ull * p);
        uint32_t sa = slot, acc = 0x1102f9u; // f9 02 11 pending (FILL = 3)
#define PC(S) push_child<S>(sa, acc, ch[2 * S], ch[2 * S + 1]);
        PC(0) PC(1) PC(2) PC(3) PC(4) PC(5) PC(6) PC(7) PC(8) PC(9) PC(10) PC(11) PC(12) PC(13) PC(14) PC(15)
#undef PC
        // after 16 children: 3 + 33*16 = 531 bytes, FILL = 3: the empty value 0x80 completes the last word
        sts32(sa, acc | (0x80u << 24));
        uint64_t st[25];
#pragma unroll
        for (int k = 0; k < 25; ++k) st[k] = 0;
        absorb_full_smem<2>(st, slot);
        absorb_full_smem<2>(st, slot + 136);
        absorb_full_smem<2>(st, slot + 272);
        absorb_final_smem<2>(st, slot + 408, 532 - 408, FR_SLOT - 408);
        uint4* o = reinterpret_cast<uint4*>(level + 32ull * p);
        o[0] = make_uint4((uint32_t)st[0], (uint32_t)(st[0] >> 32), (uint32_t)st[1], (uint32_t)(st[1] >> 32));
        o[1] = make_uint4((uint32_t)st[2], (uint32_t)(st[2] >> 32), (uint32_t)st[3], (uint32_t)(st[3] >> 32));
    }
}

// Dirty leaves: rlp([hp(key nibbles [depth, 64), leaf), value]) built in the slot, hashed, stored at the leaf's position.
// Values up to FR_SLOT - 48 bytes (the caller checks); one thread per leaf.
__global__ void __launch_bounds__(FR_WARPS * 32)
frontier_leaf_kernel(const uint8_t* __restrict__ keys32, const uint8_t* __restrict__ vals, const uint32_t* __restrict__ val_off, uint32_t n,
                     uint32_t depth, uint8_t* __restrict__ leaf_level, const uint32_t* __restrict__ pos_in, const uint32_t* __restrict__ refuse)
{
    extern __shared__ __align__(16) uint8_t fr_smem[];
    const uint32_t slot = (uint32_t)__cvta_generic_to_shared(fr_smem) + threadIdx.x * FR_SLOT;
    if (*refuse) return; // duplicate leaf positions: the update is refused as a whole
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const uint8_t* key = keys32 + 32ull * k;
        const uint32_t pos = pos_in[k];
        const uint32_t cnt = 64 - depth, hpn = 1 + cnt / 2;
        const uint32_t vl = val_off[k + 1] - val_off[k];
        const uint8_t* v = vals + val_off[k];
        const uint32_t s_hp = hpn == 1 ? 1 : 1 + hpn, s_v = (uint32_t)str_size(vl, vl ? v[0] : 0);
        const uint32_t payload = s_hp + s_v;
        uint32_t sa = slot;
        if (payload <= 55) { sts8(sa++, 0xc0 + payload); }
        else if (payload < 256) { sts8(sa++, 0xf8); sts8(sa++, payload); }
        else { sts8(sa++, 0xf9); sts8(sa++, payload >> 8); sts8(sa++, payload & 255); }
        if (hpn > 1) sts8(sa++, 0x80 + hpn);
        uint32_t i = depth;
#define KN(j) (((j) & 1) ? (key[(j) >> 1] & 15u) : (key[(j) >> 1] >> 4))
        if (cnt & 1) { sts8(sa++, 0x30 | KN(i)); ++i; } else sts8(sa++, 0x20);
        for (; i < 64; i += 2) sts8(sa++, (KN(i) << 4) | KN(i + 1));
#undef KN
        if (s_v > vl) {
            if (vl <= 55) sts8(sa++, 0x80 + vl);
            else if (vl < 256) { sts8(sa++, 0xb8); sts8(sa++, vl); }
            else { sts8(sa++, 0xb9); sts8(sa++, vl >> 8); sts8(sa++, vl & 255); }
        }
        for (uint32_t b = 0; b < vl; ++b) sts8(sa++, v[b]);
        const uint32_t len = sa - slot;
        uint64_t st[25];
#pragma unroll
        for (int q = 0; q < 25; ++q) st[q] = 0;
        uint32_t at = slot, rem = len;
        while (rem >= 136) { absorb_full_smem<2>(st, at); at += 136; rem -= 136; }
        absorb_final_smem<2>(st, at, rem, slot + FR_SLOT - at);
        uint4* o = reinterpret_cast<uint4*>(leaf_level + 32ull * pos);
        o[0] = make_uint4((uint32_t)st[0], (uint32_t)(st[0] >> 32), (uint32_t)st[1], (uint32_t)(st[1] >> 32));
        o[1] = make_uint4((uint32_t)st[2], (uint32_t)(st[2] >> 32), (uint32_t)st[3], (uint32_t)(st[3] >> 32));
    }
}

// sorted leaf positions: two dirty keys on one leaf position (a repeated key, or keys sharing their first `depth` nibbles)
// would race on leaf_level[pos]; flag it so that every later kernel of the update leaves the trie untouched
__global__ void ctrie_dup_check_kernel(const uint32_t* __restrict__ sorted_pos, uint64_t n, uint32_t* __restrict__ flag)
{
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k + 1 < n; k += (uint64_t)gridDim.x * blockDim.x)
        if (sorted_pos[k] == sorted_pos[k + 1]) *flag = 1;
}

// children (sorted, `*count` valid of `bound`) -> parents = children >> 4, the tail padded with the last valid value so
// that a fixed-size Unique over `bound` items yields exactly the distinct parents without the host knowing `*count`
__global__ void shift4_pad_kernel(const uint32_t* __restrict__ in, const uint32_t* __restrict__ count_ptr, uint32_t bound, uint32_t* __restrict__ out)
{
    uint32_t count = *count_ptr;
    if (count > bound) count = bound;
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < bound; k += gridDim.x * blockDim.x)
        out[k] = count ? in[k < count ? k : count - 1] >> 4 : 0;
}

} // namespace

// ------------------------------------------------------------------------------------------------
// U kind 1: a SPARSE resident secure trie (32-byte keys, arbitrary values) -- the structure behind StateDB.root() for a real
// state (hook src/blockchain/blockchain.zig:83-85): after a block only the dirty part is re-hashed.
//
// Resident on the device:  the sorted row table (KRow: key, value offset and length into an append-only value arena, leaf-
// reference cache), and a DENSE TOP of L nibble levels: level d holds the 16^d node references of depth d.  Level L's entries
// are the roots of the 16^L BUCKETS -- the sparse subtrees of the keys sharing an L-nibble prefix.  Keys are Keccak
// outputs, so with 16..256 keys per bucket (L = floor(log16(n / 16))) every node above the buckets is a real branch with
// >= 2 children and needs no extension / collapse logic; this is CHECKED on the device at every update, and when it does
// not hold (adversarial or tiny key sets) L is lowered and the top rebuilt -- L = 0 is one bucket = a plain rebuild.
//
// An update (upserts; an empty value deletes): sort the dirty keys into dirty rows, merge them into the table (positions by
// lower bound + two scans, the scheme the world state's tables share), re-build ONLY the dirty buckets as one forest with
// the M builder (build_forest with start_depth = L: leaves, extensions, embedded nodes and all of mptize's rules apply inside
// a bucket), then re-hash the dirty frontier of the L dense levels bottom-up (one launch per level, variable child masks).
// Pure value updates skip the merge.
// ------------------------------------------------------------------------------------------------
struct SRec { uint64_t off; uint32_t len; uint32_t pad; };
// the key first, so that row_cmp<32> / row_lower_bound apply; cache = [leaf_start + 1 (0 = nothing cached)] + the 32-byte
// digest of the key's leaf as it was last encoded (leaf_cache_probe_kernel)
struct alignas(16) KRow { uint8_t key[32]; uint64_t off; uint32_t len; uint8_t cache[33]; };
static_assert(sizeof(KRow) == 80, "row layout");

struct SparseTrie {
    uint64_t n = 0;
    DevBuf rows[2];          // the sorted row table, ping-pong across merges
    int cur = 0;
    DevBuf arena;
    uint64_t arena_used = 0;
    uint32_t L = 0;
    DevBuf top, present;     // levels 0..L: 32-byte reference + presence byte per node; level d starts at node (16^d - 1) / 15
    DevBuf dirty, buckets, gather, gvals, sort; // scratch: strie_dirty_area; st_rebuild's per-bucket and per-key gathers; the sort
    uint8_t root[32];
    uint64_t updates = 0, rebuilds = 0;
    bool compact = false;    // keep the value arena within twice the largest possible live size (values <= compact_row bytes)
    uint32_t compact_row = 0;
};

namespace {

// first node of dense level d
constexpr uint64_t level_base(uint32_t d) { return ((1ull << (4 * d)) - 1) / 15; }
// dense depth for n keys: 16 .. 255 keys per bucket
constexpr uint32_t st_target_L(uint32_t n)
{
    uint32_t L = 0;
    while (L < 6 && (n >> (4 * (L + 1))) >= 16) ++L;
    return L;
}

__device__ __forceinline__ int cmp_key32(const uint8_t* a, const uint8_t* b)
{
    const uint4 a0 = *reinterpret_cast<const uint4*>(a), a1 = *reinterpret_cast<const uint4*>(a + 16);
    const uint4 b0 = *reinterpret_cast<const uint4*>(b), b1 = *reinterpret_cast<const uint4*>(b + 16);
    const uint32_t aw[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w}, bw[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t x = __byte_perm(aw[i], 0, 0x0123), y = __byte_perm(bw[i], 0, 0x0123); // big-endian order
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}
__device__ __forceinline__ uint32_t key_prefix(const uint8_t* key, uint32_t L) // first L <= 7 nibbles as an integer
{
    const uint32_t w = __byte_perm(*reinterpret_cast<const uint32_t*>(key), 0, 0x0123);
    return L ? w >> (32 - 4 * L) : 0;
}

// ---- merging sorted dirty rows into a sorted table of rows that start with a KB-byte key: kind 1's table, and the world
// state's slot table and account rows ----
template <int KB> __device__ __forceinline__ int row_cmp(const uint8_t* a, const uint8_t* b)
{
    const int c = cmp_key32(a, b);
    return (KB == 32 || c) ? c : cmp_key32(a + 32, b + 32);
}
template <class Row, int KB> __device__ uint32_t row_lower_bound(const Row* t, uint32_t n, const uint8_t* q)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (row_cmp<KB>((const uint8_t*)(t + mid), q) < 0) a = mid + 1; else b = mid;
    }
    return a;
}
template <class Row, int KB>
__global__ void rs_classify_kernel(const Row* __restrict__ table, uint32_t n, const Row* __restrict__ dirty, uint32_t m, const uint8_t* __restrict__ del,
                                   const uint8_t* __restrict__ absent /*nullable*/, uint32_t* __restrict__ lb,
                                   uint8_t* __restrict__ kind /*0 no-op, 1 found, 2 insert, 3 delete*/, uint32_t* __restrict__ del_flag,
                                   uint32_t* __restrict__ ins_at, uint32_t* __restrict__ ins_flag, uint32_t* __restrict__ counters /*[0] ins, [1] del*/)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint8_t* q = (const uint8_t*)(dirty + j);
        const uint32_t a = row_lower_bound<Row, KB>(table, n, q);
        const bool found = a < n && row_cmp<KB>((const uint8_t*)(table + a), q) == 0 && !(absent && absent[j]);
        const uint8_t k = found ? (del[j] ? 3 : 1) : (del[j] ? 0 : 2);
        lb[j] = a;
        kind[j] = k;
        ins_flag[j] = k == 2;
        if (k == 3) { del_flag[a] = 1; atomicAdd(&counters[1], 1u); }
        if (k == 2) { atomicAdd(&ins_at[a], 1u); atomicAdd(&counters[0], 1u); }
    }
}
template <class Row>
__global__ void rs_merge_table_kernel(const Row* __restrict__ table, uint32_t n, const uint32_t* __restrict__ del_flag, const uint32_t* __restrict__ K,
                                      const uint32_t* __restrict__ I, Row* __restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (!del_flag[i]) out[K[i] + I[i + 1]] = table[i];
}
template <class Row>
__global__ void rs_merge_dirty_kernel(const Row* __restrict__ dirty, const uint8_t* __restrict__ kind, const uint32_t* __restrict__ lb,
                                      const uint32_t* __restrict__ ins_index, uint32_t m, const uint32_t* __restrict__ K, Row* __restrict__ out)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x)
        if (kind[j] == 2) out[K[lb[j]] + ins_index[j]] = dirty[j];
}
template <class Row>
__global__ void rs_replace_kernel(const Row* __restrict__ dirty, const uint8_t* __restrict__ kind, const uint32_t* __restrict__ lb, uint32_t m,
                                  Row* __restrict__ table)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x)
        if (kind[j] == 1) table[lb[j]] = dirty[j];
}
__global__ void st_keep_kernel(const uint32_t* __restrict__ del_flag, uint32_t n, uint32_t* __restrict__ keep /*n+1, keep[n] = 0*/)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) keep[i] = i < n && !del_flag[i] ? 1 : 0;
}

// Kind 1's dirty rows, in key order: key, value length, no cached leaf reference, and the value's arena offset -- the staged
// values are appended to the arena as one block, in the order given, so it is known before classification.  An empty value
// deletes.
__global__ void st_dirty_rows_kernel(const uint8_t* __restrict__ keys, const uint32_t* __restrict__ val_off, const uint32_t* __restrict__ perm,
                                     uint32_t m, uint64_t arena_base, KRow* __restrict__ rows, uint8_t* __restrict__ del,
                                     uint32_t* __restrict__ counters /*[2] duplicate key*/)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint32_t i = perm[j];
        KRow& r = rows[j];
        const uint4* s = reinterpret_cast<const uint4*>(keys + 32ull * i);
        uint4* d = reinterpret_cast<uint4*>(r.key);
        d[0] = s[0]; d[1] = s[1];
        const uint32_t len = val_off[i + 1] - val_off[i];
        r.off = arena_base + val_off[i] - val_off[0];
        r.len = len;
        r.cache[0] = 0;
        del[j] = len == 0;
        if (j + 1 < m && cmp_key32(keys + 32ull * i, keys + 32ull * perm[j + 1]) == 0) counters[2] = 1;
    }
}
// bucket of each dirty row + "first of its bucket" flag
__global__ void st_bucket_flag_kernel(const KRow* __restrict__ rows, uint32_t m, uint32_t L, uint32_t* __restrict__ bucket, uint32_t* __restrict__ first)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint32_t b = key_prefix(rows[j].key, L);
        bucket[j] = b;
        first[j] = j == 0 || key_prefix(rows[j - 1].key, L) != b;
    }
}
__global__ void st_compact_kernel(const uint32_t* __restrict__ val, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, uint32_t m,
                                  uint32_t* __restrict__ out)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x)
        if (flag[j]) out[pos[j]] = val[j];
}
// table range of each listed bucket (nullptr list = bucket u itself)
__global__ void st_bucket_range_kernel(const KRow* __restrict__ table, uint32_t n, uint32_t L, const uint32_t* __restrict__ list, uint32_t nb,
                                       uint32_t* __restrict__ lo_out, uint32_t* __restrict__ cnt_out)
{
    for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < nb; u += gridDim.x * blockDim.x) {
        const uint32_t b = list ? list[u] : u;
        uint32_t r[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const uint32_t want = b + e;
            uint32_t lo = 0, hi = n;
            if (L == 0) lo = e ? n : 0;
            else while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (key_prefix(table[mid].key, L) < want) lo = mid + 1; else hi = mid;
            }
            r[e] = lo;
        }
        lo_out[u] = r[0];
        cnt_out[u] = r[1] - r[0];
    }
}
// gather the keys of the listed buckets into a contiguous forest input (warp per bucket)
__global__ void st_gather_keys_kernel(const KRow* __restrict__ table, const uint32_t* __restrict__ lo, const uint32_t* __restrict__ seg_off, uint32_t nb,
                                      uint8_t* __restrict__ gkeys, uint32_t* __restrict__ gkey_off, uint32_t* __restrict__ seg_of_key,
                                      uint64_t* __restrict__ gval_size, SRec* __restrict__ grec, uint8_t* __restrict__ gcache)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < nb; u += warps) {
        const uint32_t base = seg_off[u], cnt = seg_off[u + 1] - base, from = lo[u];
        for (uint32_t t = lane; t < cnt; t += 32) {
            const KRow& r = table[from + t];
            const uint4* s = reinterpret_cast<const uint4*>(r.key);
            uint4* d = reinterpret_cast<uint4*>(gkeys + 32ull * (base + t));
            d[0] = s[0]; d[1] = s[1];
            gkey_off[base + t] = 32u * (base + t);
            seg_of_key[base + t] = u;
            gval_size[base + t] = r.len;
            grec[base + t] = SRec{r.off, r.len, 0};
            uint8_t* g = gcache + 33ull * (base + t);
            const uint32_t* cw = reinterpret_cast<const uint32_t*>(r.cache); // 4-byte aligned in KRow: 8 word loads + 1 byte
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                const uint32_t x = cw[w];
                g[4 * w] = x; g[4 * w + 1] = x >> 8; g[4 * w + 2] = x >> 16; g[4 * w + 3] = x >> 24;
            }
            g[32] = r.cache[32];
        }
    }
}
// the leaf references of this build back into the table's rows
__global__ void st_scatter_cache_kernel(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ seg_off, uint32_t nb, const uint8_t* __restrict__ gcache_out,
                                        KRow* __restrict__ table)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < nb; u += warps) {
        const uint32_t base = seg_off[u], cnt = seg_off[u + 1] - base, from = lo[u];
        for (uint32_t t = lane; t < cnt; t += 32) {
            const uint8_t* g = gcache_out + 33ull * (base + t);
            KRow& r = table[from + t];
            uint32_t* cw = reinterpret_cast<uint32_t*>(r.cache); // 4-byte aligned in KRow: 8 word stores + 1 byte
#pragma unroll
            for (int w = 0; w < 8; ++w) cw[w] = g[4 * w] | (uint32_t)g[4 * w + 1] << 8 | (uint32_t)g[4 * w + 2] << 16 | (uint32_t)g[4 * w + 3] << 24;
            r.cache[32] = g[32];
        }
    }
}
// values into a contiguous buffer at gval_off (Rec: the gathered records of a rebuild, or the table's rows)
template <class Rec>
__global__ void st_gather_vals_kernel(const uint8_t* __restrict__ arena, const Rec* __restrict__ grec, const uint64_t* __restrict__ gval_off, uint32_t mk,
                                      uint8_t* __restrict__ gvals)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < mk; t += warps) {
        const uint64_t src = grec[t].off, dst = gval_off[t];
        const uint32_t len = grec[t].len;
        for (uint32_t b = lane; b < len; b += 32) gvals[dst + b] = arena[src + b];
    }
}
__global__ void st_scatter_roots_kernel(const uint8_t* __restrict__ roots, const uint32_t* __restrict__ list, const uint32_t* __restrict__ cnt, uint32_t nb,
                                        uint8_t* __restrict__ level, uint8_t* __restrict__ present)
{
    for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < nb; u += gridDim.x * blockDim.x) {
        const uint32_t b = list ? list[u] : u;
        const uint4* s = reinterpret_cast<const uint4*>(roots + 32ull * u);
        uint4* d = reinterpret_cast<uint4*>(level + 32ull * b);
        d[0] = s[0]; d[1] = s[1];
        present[b] = cnt[u] ? 1 : 0;
    }
}
// the number of valid children stays on the device (*cnt_ptr <= bound): no host read-back per dense level
__global__ void st_parent_flag_kernel(const uint32_t* __restrict__ child, const uint32_t* __restrict__ cnt_ptr, uint32_t bound, uint32_t* __restrict__ parent,
                                      uint32_t* __restrict__ first)
{
    const uint32_t cnt = *cnt_ptr < bound ? *cnt_ptr : bound;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j <= bound; j += gridDim.x * blockDim.x) {
        if (j < cnt) {
            parent[j] = child[j] >> 4;
            first[j] = j == 0 || (child[j - 1] >> 4) != (child[j] >> 4);
        } else first[j] = 0;
    }
}
// One dense-top node per thread: rlp([ref or "" x 16, ""]) over the children that exist (src/mpt/mpt.zig:218-247), built in the
// thread's shared-memory slot, hashed with the product sponge.  A node with exactly ONE child would have to collapse into
// an extension / its child (mpt.zig:83-106): that breaks the dense-top premise and is reported through violation[owner].
// Many tries' dense tops can share one pool: listed node i then sits at level[bases[i] + p], its children at
// child_level[bases[i] + 16p + v], and owners[i] says which violation flag it reports to.
__global__ void __launch_bounds__(FR_WARPS * 32)
st_top_branch_kernel(const uint8_t* __restrict__ child_level, const uint8_t* __restrict__ child_present, const uint32_t* __restrict__ parents /*nullable*/,
                     const uint32_t* __restrict__ bases /*nullable: all 0*/, const uint32_t* __restrict__ owners /*nullable: all 0*/,
                     uint32_t count, const uint32_t* __restrict__ count_ptr /*nullable: the count lives on the device, `count` is its bound*/,
                     uint8_t* __restrict__ level, uint8_t* __restrict__ present, uint32_t* __restrict__ violation)
{
    extern __shared__ __align__(16) uint8_t fr_smem[];
    const uint32_t slot = (uint32_t)__cvta_generic_to_shared(fr_smem) + threadIdx.x * FR_SLOT;
    if (count_ptr && *count_ptr < count) count = *count_ptr;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const uint64_t base = bases ? bases[i] : 0;
        const uint64_t p = (parents ? parents[i] : i) + base, c0 = 16ull * (p - base) + base; // this node; its first child
        uint32_t mask = 0;
        for (uint32_t v = 0; v < 16; ++v) mask |= (child_present[c0 + v] ? 1u : 0u) << v;
        const uint32_t c = __popc(mask);
        if (c == 0) { present[p] = 0; continue; }
        if (c == 1) atomicExch(violation + (owners ? owners[i] : 0), 1u);
        present[p] = 1;
        const uint32_t payload = 33 * c + (16 - c) + 1;
        uint32_t sa = slot;
        if (payload <= 55) sts8(sa++, 0xc0 + payload);
        else if (payload < 256) { sts8(sa++, 0xf8); sts8(sa++, payload); }
        else { sts8(sa++, 0xf9); sts8(sa++, payload >> 8); sts8(sa++, payload & 255); }
        for (uint32_t v = 0; v < 16; ++v) {
            if (!((mask >> v) & 1)) { sts8(sa++, 0x80); continue; }
            sts8(sa++, 0xa0);
            const uint4* h = reinterpret_cast<const uint4*>(child_level + 32ull * (c0 + v));
            const uint4 a = h[0], b = h[1];
            const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
            for (int k = 0; k < 8; ++k) { sts8(sa++, w[k] & 255); sts8(sa++, (w[k] >> 8) & 255); sts8(sa++, (w[k] >> 16) & 255); sts8(sa++, w[k] >> 24); }
        }
        sts8(sa++, 0x80);
        const uint32_t len = sa - slot;
        uint64_t st[25];
#pragma unroll
        for (int q = 0; q < 25; ++q) st[q] = 0;
        uint32_t at = slot, rem = len;
        while (rem >= 136) { absorb_full_smem<2>(st, at); at += 136; rem -= 136; }
        absorb_final_smem<2>(st, at, rem, slot + FR_SLOT - at);
        uint4* o = reinterpret_cast<uint4*>(level + 32ull * p);
        o[0] = make_uint4((uint32_t)st[0], (uint32_t)(st[0] >> 32), (uint32_t)st[1], (uint32_t)(st[1] >> 32));
        o[1] = make_uint4((uint32_t)st[2], (uint32_t)(st[2] >> 32), (uint32_t)st[3], (uint32_t)(st[3] >> 32));
    }
}

// The frontier kernels' FR_SMEM bytes of dynamic shared memory exceed the 48 KB default: opt in once per device (function
// attributes are per device, as launch_staged in keccak_kernels.cu)
int fr_opt_in(phant_gpu_ctx* ctx)
{
    static bool attr[64] = {false};
    bool& opted = attr[(ctx->device >= 0 && ctx->device < 64) ? ctx->device : 0];
    if (opted) return PHANT_GPU_OK;
    for (const void* f : {(const void*)frontier_leaf_kernel, (const void*)frontier_branch_kernel, (const void*)st_top_branch_kernel})
        CU(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, FR_SMEM));
    opted = true;
    return PHANT_GPU_OK;
}
// a frontier kernel's grid for `items` threads, capped at 3 CTAs per SM (the kernels loop over the rest)
unsigned fr_grid(int dev, uint64_t items)
{
    const uint64_t g = (items + FR_WARPS * 32 - 1) / (FR_WARPS * 32), cap = (uint64_t)keccak_num_sms(dev) * 3;
    return (unsigned)(g < cap ? g : cap);
}

// merge sorted dirty rows (classified) into table[cur] -> table[1 - cur]; `n_new` rows result
template <class Row>
int rs_merge(phant_gpu_ctx* ctx, DevBuf* table, int& cur, uint32_t n, const Row* dirty, uint32_t m, const uint8_t* kind,
             const uint32_t* lb, const uint32_t* ins_flag, uint32_t* del_flag, uint32_t* ins_at, uint32_t* keep, uint32_t* K, uint32_t* I,
             uint32_t* ins_index)
{
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device, nxt = 1 - cur;
    st_keep_kernel<<<grid1d(dev, n + 1, 256), 256, 0, s>>>(del_flag, n, keep);
    RC(scan_u32(ctx, keep, K, n + 1));
    RC(scan_u32(ctx, ins_at, I, n + 2));
    if (m) RC(scan_u32(ctx, ins_flag, ins_index, m));
    if (n) rs_merge_table_kernel<Row><<<grid1d(dev, n, 256), 256, 0, s>>>((const Row*)table[cur].ptr, n, del_flag, K, I, (Row*)table[nxt].ptr);
    if (m) rs_merge_dirty_kernel<Row><<<grid1d(dev, m, 256), 256, 0, s>>>(dirty, kind, lb, ins_index, m, K, (Row*)table[nxt].ptr);
    ctx->stats.launches += 6;
    cur = nxt;
    return PHANT_GPU_OK;
}

// The counter words of a sparse trie update, in the context's sp_words: strie_apply's classification counts and st_rebuild's
// dense-level words.  They are not in the trie's own areas, whose sizes the world state reports as its device_bytes.
struct SpWords {
    uint32_t* classify; // [0] inserts, [1] deletes, [2] a key twice
    uint32_t* viol;     // a dense node with fewer than two children
    uint32_t* parents;  // the current dense level's parent count
};
int sp_words(phant_gpu_ctx* ctx, SpWords* w)
{
    return carve(ctx, ctx->sp_words, [&](Carve& c) { w->classify = c.take<uint32_t>(4); w->viol = c.take<uint32_t>(1); w->parents = c.take<uint32_t>(1); });
}

// (re)build the listed buckets (d_list == nullptr: all 16^L of them) and the dense levels above them; root -> sp.root
int st_rebuild(phant_gpu_ctx* ctx, SparseTrie& sp, const uint32_t* d_list, uint32_t nb, bool all)
{
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t L = sp.L, n = (uint32_t)sp.n;
    KRow* table = (KRow*)sp.rows[sp.cur].ptr;
    uint8_t* top = (uint8_t*)sp.top.ptr;
    uint8_t* pres = (uint8_t*)sp.present.ptr;
    if (n == 0) { memcpy(sp.root, EMPTY_ROOT_H, 32); return PHANT_GPU_OK; }
    PhaseTrace tr(s);
    // per bucket: table range, size, root; per dense node: parent lists
    uint32_t *lo, *cnt, *seg_off, *par, *flag, *pos, *ping[2];
    uint8_t* roots;
    RC(carve(ctx, sp.buckets, [&](Carve& c) {
        lo = c.take<uint32_t>(nb + 2); cnt = c.take<uint32_t>(nb + 2); seg_off = c.take<uint32_t>(nb + 2); roots = c.take<uint8_t>(32ull * nb);
        par = c.take<uint32_t>(nb + 2); flag = c.take<uint32_t>(nb + 2); pos = c.take<uint32_t>(nb + 2); // parents, first-of-parent flags, positions
        ping[0] = c.take<uint32_t>(nb + 2); ping[1] = c.take<uint32_t>(nb + 2);                           // two parent lists
    }));
    st_bucket_range_kernel<<<grid1d(dev, nb, 128), 128, 0, s>>>(table, n, L, d_list, nb, lo, cnt);
    CU(cudaMemsetAsync(cnt + nb, 0, 4, s));
    RC(scan_u32(ctx, cnt, seg_off, nb + 1));
    uint32_t mk = 0;
    CU(cudaMemcpyAsync(&mk, seg_off + nb, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    if (mk) {
        uint8_t *gkeys, *gcache, *gcache_out;
        uint32_t *gkoff, *seg_of_key;
        uint64_t *gsize, *gvoff;
        SRec* grec;
        RC(carve(ctx, sp.gather, [&](Carve& g) {
            gkeys = g.take<uint8_t>(32ull * mk); gkoff = g.take<uint32_t>(mk + 2); seg_of_key = g.take<uint32_t>(mk + 2);
            gsize = g.take<uint64_t>(mk + 2); gvoff = g.take<uint64_t>(mk + 2); grec = g.take<SRec>(mk);
            gcache = g.take<uint8_t>(33ull * mk); gcache_out = g.take<uint8_t>(33ull * mk);
        }));
        st_gather_keys_kernel<<<grid1d(dev, nb, 256, 32), 256, 0, s>>>(table, lo, seg_off, nb, gkeys, gkoff, seg_of_key, gsize, grec, gcache);
        const uint32_t last = 32u * mk;
        CU(cudaMemcpyAsync(gkoff + mk, &last, 4, cudaMemcpyHostToDevice, s));
        RC(scan_sizes(ctx, gsize, gvoff, mk));
        uint64_t vbytes = 0;
        CU(cudaMemcpyAsync(&vbytes, gvoff + mk, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        RC(sp.gvals.reserve(ctx, vbytes + 64));
        st_gather_vals_kernel<<<grid1d(dev, mk, 256, 32), 256, 0, s>>>((const uint8_t*)sp.arena.ptr, grec, gvoff, mk, (uint8_t*)sp.gvals.ptr);
        ctx->stats.launches += 3;
        tr.mark("  bucket ranges + gathers");
        RC(build_forest(ctx, {.keys = gkeys, .key_off = gkoff, .vals = (const uint8_t*)sp.gvals.ptr, .val_off = gvoff, .n = mk, .seg_off = seg_off,
                              .n_seg = nb, .seg_of_key = seg_of_key, .roots = roots, .start_depth = L, .leaf_cache = gcache, .leaf_cache_out = gcache_out}));
        tr.mark("  build_forest");
        st_scatter_cache_kernel<<<grid1d(dev, nb, 256, 32), 256, 0, s>>>(lo, seg_off, nb, gcache_out, table);
        ctx->stats.launches++;
    }
    if (L == 0) { // one bucket: its root is the trie's root
        CU(cudaMemcpyAsync(sp.root, roots, 32, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        return PHANT_GPU_OK;
    }
    st_scatter_roots_kernel<<<grid1d(dev, nb, 256), 256, 0, s>>>(roots, d_list, cnt, nb, top + 32 * level_base(L), pres + level_base(L));
    ctx->stats.launches++;
    // dense levels bottom-up: parents of the dirty children
    RC(fr_opt_in(ctx));
    SpWords words;
    RC(sp_words(ctx, &words));
    uint32_t* viol = words.viol;
    CU(cudaMemsetAsync(viol, 0, 4, s));
    const uint32_t* child = d_list;
    uint32_t cbound = nb;                       // upper bound of the children count; the exact count stays on the device
    uint32_t* cnt_dev = words.parents;
    CU(cudaMemcpyAsync(cnt_dev, &nb, 4, cudaMemcpyHostToDevice, s));
    for (int d = (int)L - 1; d >= 0; --d) {
        const uint32_t* plist = nullptr;
        uint32_t pbound = 1u << (4 * d);
        const uint32_t* pcount_dev = nullptr;
        if (!all) { // distinct parents of the (sorted) dirty children
            uint32_t* uniq = ping[d & 1];
            st_parent_flag_kernel<<<grid1d(dev, cbound + 1, 256), 256, 0, s>>>(child, cnt_dev, cbound, par, flag);
            RC(scan_u32(ctx, flag, pos, cbound + 1));
            st_compact_kernel<<<grid1d(dev, cbound, 256), 256, 0, s>>>(par, flag, pos, cbound, uniq);
            CU(cudaMemcpyAsync(cnt_dev, pos + cbound, 4, cudaMemcpyDeviceToDevice, s)); // the parents are the next level's children
            if (cbound < pbound) pbound = cbound;
            plist = uniq;
            child = uniq;
            cbound = pbound;
            pcount_dev = cnt_dev;
            ctx->stats.launches += 3;
        }
        st_top_branch_kernel<<<fr_grid(dev, pbound), FR_WARPS * 32, FR_SMEM, s>>>(top + 32 * level_base(d + 1), pres + level_base(d + 1), plist, nullptr, nullptr,
                                                                                pbound, pcount_dev,
                                                                                top + 32 * level_base(d), pres + level_base(d), viol);
        ctx->stats.launches++;
    }
    CU(cudaGetLastError());
    tr.mark("  dense levels");
    uint32_t v = 0;
    CU(cudaMemcpyAsync(sp.root, top, 32, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&v, viol, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return v ? 1 : PHANT_GPU_OK; // 1 = the dense-top premise does not hold at this L
}

int st_set_L_and_rebuild_all(phant_gpu_ctx* ctx, SparseTrie& sp, uint32_t L)
{
    for (;;) {
        sp.L = L;
        const uint64_t nodes = level_base(L + 1);
        RC(sp.top.reserve(ctx, 32 * nodes + 64));
        RC(sp.present.reserve(ctx, nodes + 64));
        CU(cudaMemsetAsync(sp.present.ptr, 0, nodes, ctx->stream));
        sp.rebuilds++;
        const int rc = st_rebuild(ctx, sp, nullptr, 1u << (4 * L), true);
        if (rc != 1) return rc;
        if (L == 0) return PHANT_GPU_E_CUDA; // cannot happen: L = 0 has no dense level
        --L; // some top node has a single child: fewer dense levels
    }
}

// Everything an update of m keys with vb value bytes works in (sp.dirty), laid out in one place so that a caller can reserve
// it before its first write: the staging area the caller fills on the device (the dirty keys as given, the values, their
// m+1 offsets), the sorted dirty rows with their classification, and the merge scratch of the n-row table.
struct StrieDirty {
    uint8_t* keys; uint8_t* vals; uint32_t* val_off;
    uint32_t* perm; KRow* rows; uint8_t* del; uint8_t* kind;
    uint32_t *lb, *ins_flag, *ins_index, *bucket;
    uint32_t *del_flag, *ins_at, *keep, *K, *I;
};
int strie_dirty_area(phant_gpu_ctx* ctx, SparseTrie& sp, uint32_t m, uint64_t vb, StrieDirty* a)
{
    const uint64_t n = sp.n;
    RC(carve(ctx, sp.dirty, [&](Carve& c) {
        a->keys = c.take<uint8_t>(32ull * m);
        a->vals = c.take<uint8_t>(vb);
        a->val_off = c.take<uint32_t>(m + 1);
        a->perm = c.take<uint32_t>(m);
        a->rows = c.take<KRow>(m);
        a->del = c.take<uint8_t>(m);
        a->kind = c.take<uint8_t>(m);
        a->lb = c.take<uint32_t>(m);
        a->ins_flag = c.take<uint32_t>(m + 1);
        a->ins_index = c.take<uint32_t>(m + 1);
        a->bucket = c.take<uint32_t>(m);
        a->del_flag = c.take<uint32_t>((n + 3) * 5); // del_flag and ins_at first: one memset clears both
    }));
    a->ins_at = a->del_flag + n + 3;
    a->keep = a->ins_at + n + 3;
    a->K = a->keep + n + 3;
    a->I = a->K + n + 3;
    return PHANT_GPU_OK;
}

__global__ void st_rec_len_kernel(const KRow* __restrict__ rows, uint32_t n, uint64_t* __restrict__ len)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) len[i] = rows[i].len;
}
__global__ void st_rebase_recs_kernel(KRow* __restrict__ rows, uint32_t n, const uint64_t* __restrict__ off)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) rows[i].off = off[i];
}

// Copy the live values (table order) into a fresh arena sized for twice the largest live size n * compact_row.
int strie_compact_arena(phant_gpu_ctx* ctx, SparseTrie& sp)
{
    cudaStream_t s = ctx->stream;
    const uint32_t n = (uint32_t)sp.n;
    KRow* rows = (KRow*)sp.rows[sp.cur].ptr;
    uint64_t *len, *off;
    RC(carve(ctx, sp.gather, [&](Carve& c) { len = c.take<uint64_t>(n + 1); off = c.take<uint64_t>(n + 1); }));
    st_rec_len_kernel<<<grid1d(ctx->device, n, 256), 256, 0, s>>>(rows, n, len);
    RC(scan_sizes(ctx, len, off, n));
    uint64_t live = 0;
    CU(cudaMemcpyAsync(&live, off + n, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    DevBuf fresh;
    RC(fresh.reserve(ctx, 2ull * sp.compact_row * n + (1 << 20)));
    st_gather_vals_kernel<<<grid1d(ctx->device, n, 256, 32), 256, 0, s>>>((const uint8_t*)sp.arena.ptr, rows, off, n, (uint8_t*)fresh.ptr);
    st_rebase_recs_kernel<<<grid1d(ctx->device, n, 256), 256, 0, s>>>(rows, n, off);
    ctx->stats.launches += 4;
    CU(cudaStreamSynchronize(s));
    sp.arena.release();
    sp.arena = fresh;
    sp.arena_used = live;
    return PHANT_GPU_OK;
}

// The update itself, from the staged dirty area (strie_dirty_area), which the caller filled on the device.
int strie_apply(phant_gpu_ctx* ctx, SparseTrie& sp, uint32_t m, uint64_t vb, uint8_t out_root[32])
{
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    if (m == 0) { memcpy(out_root, sp.root, 32); return PHANT_GPU_OK; }
    const uint32_t n = (uint32_t)sp.n;
    StrieDirty a;
    RC(strie_dirty_area(ctx, sp, m, vb, &a));
    PhaseTrace tr(s);
    RC(sort_by_segment_and_hash(ctx, a.keys, nullptr, m, a.perm, sp.sort));
    tr.mark("sort dirty keys");
    // ---- dirty rows, classified against the table ----
    CU(cudaMemsetAsync(a.del_flag, 0, 4ull * (n + 3) * 2, s));
    SpWords words;
    RC(sp_words(ctx, &words));
    uint32_t* counters = words.classify;
    CU(cudaMemsetAsync(counters, 0, 16, s));
    st_dirty_rows_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(a.keys, a.val_off, a.perm, m, sp.arena_used, a.rows, a.del, counters);
    KRow* table = (KRow*)sp.rows[sp.cur].ptr;
    rs_classify_kernel<KRow, 32><<<grid1d(dev, m, 128), 128, 0, s>>>(table, n, a.rows, m, a.del, nullptr, a.lb, a.kind, a.del_flag, a.ins_at, a.ins_flag,
                                                                     counters);
    uint32_t hc[4] = {0, 0, 0, 0}, v0 = 0;
    CU(cudaMemcpyAsync(hc, counters, 16, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&v0, a.val_off, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    tr.mark("classify + readback");
    if (hc[2]) return PHANT_GPU_E_INVALID; // the same key twice in one update
    const uint32_t n_ins = hc[0], n_del = hc[1];
    // ---- values into the arena as one block, where the rows point (grown with contents preserved; compaction is a
    // rebuild-time concern) ----
    const uint64_t app_bytes = vb - v0;
    if (sp.arena_used + app_bytes + 64 > sp.arena.cap) {
        DevBuf bigger;
        RC(bigger.reserve(ctx, (sp.arena_used + app_bytes) * 2 + (1 << 20)));
        if (sp.arena_used) CU(cudaMemcpyAsync(bigger.ptr, sp.arena.ptr, sp.arena_used, cudaMemcpyDeviceToDevice, s));
        CU(cudaStreamSynchronize(s));
        sp.arena.release();
        sp.arena = bigger;
    }
    if (app_bytes) CU(cudaMemcpyAsync((uint8_t*)sp.arena.ptr + sp.arena_used, a.vals + v0, app_bytes, cudaMemcpyDeviceToDevice, s));
    sp.arena_used += app_bytes;
    // ---- replaced rows in place (a new value: no cached leaf reference), then the merge (skipped for pure value updates) ----
    rs_replace_kernel<KRow><<<grid1d(dev, m, 256), 256, 0, s>>>(a.rows, a.kind, a.lb, m, table);
    ctx->stats.launches++;
    const uint32_t new_n = n - n_del + n_ins;
    if (n_ins || n_del) {
        RC(sp.rows[1 - sp.cur].reserve(ctx, sizeof(KRow) * new_n + 64));
        RC(rs_merge<KRow>(ctx, sp.rows, sp.cur, n, a.rows, m, a.kind, a.lb, a.ins_flag, a.del_flag, a.ins_at, a.keep, a.K, a.I, a.ins_index));
        sp.n = new_n;
    }
    tr.mark("merge");
    sp.updates++;
    if (new_n == 0) {
        sp.L = 0;
        memcpy(sp.root, EMPTY_ROOT_H, 32);
        memcpy(out_root, sp.root, 32);
        return PHANT_GPU_OK;
    }
    // ---- which part of the trie to re-hash ----
    const uint32_t Lt = st_target_L(new_n);
    int rc;
    if (Lt > sp.L || Lt + 1 < sp.L || n == 0) {
        rc = st_set_L_and_rebuild_all(ctx, sp, Lt); // the table grew / shrank past a bucket-size bound: new dense depth
    } else {
        uint32_t* first = a.ins_flag;               // (classification scratch is free again)
        uint32_t* fpos = a.ins_index;
        uint32_t* list = a.lb;
        st_bucket_flag_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(a.rows, m, sp.L, a.bucket, first);
        CU(cudaMemsetAsync(first + m, 0, 4, s));
        RC(scan_u32(ctx, first, fpos, m + 1));
        st_compact_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(a.bucket, first, fpos, m, list);
        uint32_t nb = 0;
        CU(cudaMemcpyAsync(&nb, fpos + m, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches += 3;
        rc = st_rebuild(ctx, sp, list, nb, false);
        if (rc == 1) rc = st_set_L_and_rebuild_all(ctx, sp, sp.L - 1); // a dense node lost all but one child: fewer dense levels
    }
    tr.mark("rebuild (buckets + top)");
    if (rc) return rc;
    if (sp.compact && sp.arena_used > 2ull * sp.compact_row * sp.n + (1 << 20)) RC(strie_compact_arena(ctx, sp)); // over half of it is dead
    memcpy(out_root, sp.root, 32);
    ctx->stats.d2h_bytes += 36;
    return PHANT_GPU_OK;
}

int strie_update(phant_gpu_ctx* ctx, SparseTrie& sp, const uint8_t* keys32, const uint8_t* vals, const uint32_t* val_off, uint64_t m64,
                 uint8_t out_root[32])
{
    cudaStream_t s = ctx->stream;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // host tables (it is the StateDB flattening, as S)
    if (m64 == 0) { memcpy(out_root, sp.root, 32); return PHANT_GPU_OK; }
    if (!keys32 || !val_off || m64 >= (1ull << 28) || sp.n + m64 >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    const uint32_t m = (uint32_t)m64;
    for (uint32_t i = 0; i < m; ++i)
        if (val_off[i + 1] < val_off[i]) return PHANT_GPU_E_INVALID;
    const uint64_t vb = val_off[m];
    if (vb && !vals) return PHANT_GPU_E_INVALID;
    StrieDirty area;
    RC(strie_dirty_area(ctx, sp, m, vb, &area));
    PhaseTrace tr(s);
    CU(cudaMemcpyAsync(area.keys, keys32, 32ull * m, cudaMemcpyHostToDevice, s));
    if (vb) CU(cudaMemcpyAsync(area.vals, vals, vb, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(area.val_off, val_off, 4ull * (m + 1), cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += 32ull * m + vb + 4ull * (m + 1);
    tr.mark("stage dirty (H2D)");
    return strie_apply(ctx, sp, m, vb, out_root);
}

} // namespace

extern "C" int phant_gpu_trie_open(phant_gpu_ctx* ctx, const phant_gpu_trie_desc* desc, phant_gpu_trie** out)
{
    if (!ctx || !desc || !out) return PHANT_GPU_E_INVALID;
    *out = nullptr;
    if (desc->kind == 1) { // sparse resident secure trie, initially empty
        CU(cudaSetDevice(ctx->device));
        phant_gpu_trie* t = new (std::nothrow) phant_gpu_trie();
        SparseTrie* sp = new (std::nothrow) SparseTrie();
        if (!t || !sp) { delete t; delete sp; return PHANT_GPU_E_OOM; }
        t->ctx = ctx; t->kind = 1; t->depth = 0; t->sp = sp;
        memcpy(sp->root, EMPTY_ROOT_H, 32);
        *out = t;
        return PHANT_GPU_OK;
    }
    if (desc->kind != 0 || desc->depth < 1 || desc->depth > 7) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    phant_gpu_trie* t = new (std::nothrow) phant_gpu_trie();
    if (!t) return PHANT_GPU_E_OOM;
    t->ctx = ctx;
    t->depth = desc->depth;
    t->level.resize(desc->depth + 1);
    auto lay = [&](Carve& c) { for (uint32_t l = 0; l <= desc->depth; ++l) t->level[l] = c.take<uint8_t>(32ull << (4 * l)); };
    if (int rc = carve(ctx, t->store, lay)) { delete t; return rc; }
    const uint64_t n_leaves = 1ull << (4 * desc->depth);
    ctrie_fill_leaves_kernel<<<grid1d(ctx->device, n_leaves, 256), 256, 0, ctx->stream>>>(desc->seed, n_leaves, t->level[desc->depth]);
    ctx->stats.launches++;
    // all branch levels bottom-up, one frontier_branch_kernel launch each: level l's parents are the first 16^l entries of
    // one identity list, and the kernel clamps the count word (16^(depth-1)) to 16^l
    const uint32_t n_top = (uint32_t)(n_leaves >> 4);
    DevBuf ids;
    auto levels = [&]() -> int {
        RC(ids.reserve(ctx, 4ull * n_top + 16));
        RC(fr_opt_in(ctx));
        uint32_t* counts; // counts[0] = parents; counts[8] = "refused" flag, never set here
        RC(carve(ctx, t->work, [&](Carve& c) { counts = c.take<uint32_t>(16); }));
        const uint32_t init[16] = {n_top};
        CU(cudaMemcpyAsync(counts, init, sizeof init, cudaMemcpyHostToDevice, ctx->stream));
        iota_kernel<<<grid1d(ctx->device, n_top, 256), 256, 0, ctx->stream>>>((uint32_t*)ids.ptr, n_top);
        for (int l = (int)desc->depth - 1; l >= 0; --l)
            frontier_branch_kernel<<<fr_grid(ctx->device, 1ull << (4 * l)), FR_WARPS * 32, FR_SMEM, ctx->stream>>>(
                t->level[l + 1], (const uint32_t*)ids.ptr, counts, 1u << (4 * l), t->level[l], counts + 8);
        ctx->stats.launches += 1 + desc->depth;
        CU(cudaGetLastError());
        CU(cudaStreamSynchronize(ctx->stream));
        return PHANT_GPU_OK;
    };
    if (int rc = levels()) {
        cudaStreamSynchronize(ctx->stream); // nothing in flight may still use what is released
        ids.release();
        t->work.release();
        t->store.release();
        delete t;
        return rc;
    }
    ids.release();
    *out = t;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_trie_root(phant_gpu_trie* t, uint8_t out_root[32])
{
    if (!t || !out_root) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = t->ctx;
    if (t->kind == 1) { memcpy(out_root, t->sp->root, 32); return PHANT_GPU_OK; }
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(out_root, t->level[0], 32, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_trie_update(phant_gpu_trie* t, const uint8_t* keys32, const uint8_t* leaf_vals, const uint32_t* val_off,
                                     uint64_t n_dirty, uint8_t out_root[32])
{
    if (!t || !out_root) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = t->ctx;
    CU(cudaSetDevice(ctx->device));
    if (t->kind == 1) return strie_update(ctx, *t->sp, keys32, leaf_vals, val_off, n_dirty, out_root);
    cudaStream_t s = ctx->stream;
    if (n_dirty == 0) return phant_gpu_trie_root(t, out_root);
    if (!keys32 || !val_off || n_dirty >= (1ull << 28)) return PHANT_GPU_E_INVALID;
    const uint8_t* d_keys = keys32; const uint8_t* d_vals = leaf_vals; const uint32_t* d_voff = val_off;
    uint64_t vb = 0, max_val = ~0ull;
    if (!(ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS)) {
        max_val = 0;
        for (uint64_t i = 0; i < n_dirty; ++i) {
            if (val_off[i + 1] < val_off[i]) return PHANT_GPU_E_INVALID;
            if ((uint64_t)(val_off[i + 1] - val_off[i]) > max_val) max_val = val_off[i + 1] - val_off[i];
        }
        vb = val_off[n_dirty];
        if (vb && !leaf_vals) return PHANT_GPU_E_INVALID;
        uint8_t *dk, *dv;
        uint32_t* dvo;
        RC(carve(ctx, ctx->d_msgs, [&](Carve& c) { dk = c.take<uint8_t>(32 * n_dirty); dv = c.take<uint8_t>(vb); dvo = c.take<uint32_t>(n_dirty + 1); }));
        CU(cudaMemcpyAsync(dk, keys32, 32 * n_dirty, cudaMemcpyHostToDevice, s));
        if (vb) CU(cudaMemcpyAsync(dv, leaf_vals, vb, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dvo, val_off, 4 * (n_dirty + 1), cudaMemcpyHostToDevice, s));
        ctx->stats.h2d_bytes += 32 * n_dirty + vb + 4 * (n_dirty + 1);
        d_keys = dk; d_vals = dv; d_voff = dvo;
    } else {
        CU(cudaMemcpyAsync(&vb, val_off + n_dirty, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    const uint32_t L = t->depth;
    // leaves: fused (built and hashed in shared memory) when the host has seen every value fit a slot, general (batched Keccak)
    // otherwise; branch levels: the frontier kernel either way.  The only host synchronisation of a fused update is the final
    // read of the root; the general leaf stage adds the read of its arena size.
    const bool fused = !(ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) && max_val <= FR_SLOT - 48;
    RC(fr_opt_in(ctx));
    uint32_t *counts, *pos, *cur, *tmp, *uniq; // counts[0] = valid entries of `cur`; counts[8] = "refused" flag
    uint64_t *sizes, *offs;
    uint8_t* dg;
    RC(carve(ctx, t->work, [&](Carve& c) {
        counts = c.take<uint32_t>(16);
        pos = c.take<uint32_t>(n_dirty); cur = c.take<uint32_t>(n_dirty); tmp = c.take<uint32_t>(n_dirty); uniq = c.take<uint32_t>(n_dirty);
        sizes = c.take<uint64_t>(fused ? 0 : n_dirty + 2); offs = c.take<uint64_t>(fused ? 0 : n_dirty + 2); dg = c.take<uint8_t>(fused ? 0 : 32 * n_dirty);
    }));
    uint32_t* refuse = counts + 8;
    // positions first, sorted, checked for collisions; only then is anything written to the resident levels
    ctrie_leaf_pos_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_keys, n_dirty, L, pos);
    RC(cub_call(ctx, [&](void* tmp, size_t& b) {
        return cub::DeviceRadixSort::SortKeys(tmp, b, (const uint32_t*)pos, cur, (int64_t)n_dirty, 0, 4 * (int)L, s);
    }));
    const uint32_t init[16] = {(uint32_t)n_dirty};
    CU(cudaMemcpyAsync(counts, init, sizeof init, cudaMemcpyHostToDevice, s));
    ctrie_dup_check_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(cur, n_dirty, refuse);
    ctx->stats.launches += 3;
    if (fused) {
        frontier_leaf_kernel<<<fr_grid(ctx->device, n_dirty), FR_WARPS * 32, FR_SMEM, s>>>(d_keys, d_vals, d_voff, (uint32_t)n_dirty, L, t->level[L], pos, refuse);
        ctx->stats.launches++;
    } else { // encode, hash, scatter into the leaf level; a refused update returns before the scatter
        ctrie_leaf_size_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_vals, d_voff, n_dirty, L, sizes);
        RC(scan_sizes(ctx, sizes, offs, n_dirty));
        uint64_t total = 0;
        uint32_t refused = 0;
        CU(cudaMemcpyAsync(&total, offs + n_dirty, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(&refused, refuse, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        if (refused) return PHANT_GPU_E_INVALID;
        RC(t->leaf_rlp.reserve(ctx, total + 64));
        ctrie_leaf_encode_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_keys, d_vals, d_voff, n_dirty, L, offs, (uint8_t*)t->leaf_rlp.ptr);
        ctx->stats.launches += 3;
        RC(ctx->hash_csr((const uint8_t*)t->leaf_rlp.ptr, offs, n_dirty, total, dg));
        ctrie_scatter_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(dg, pos, n_dirty, t->level[L]);
        ctx->stats.launches++;
    }
    // per level: shift/pad + unique (the distinct-parent count stays on the device) + one hash launch
    uint64_t bound = n_dirty;
    for (int l = (int)L - 1; l >= 0; --l) {
        shift4_pad_kernel<<<grid1d(ctx->device, bound, 256), 256, 0, s>>>(cur, counts, (uint32_t)bound, tmp);
        RC(cub_call(ctx, [&](void* temp, size_t& b) { return cub::DeviceSelect::Unique(temp, b, (const uint32_t*)tmp, uniq, counts, (int64_t)bound, s); }));
        if (bound > (1ull << (4 * l))) bound = 1ull << (4 * l); // a level cannot have more dirty nodes than nodes
        frontier_branch_kernel<<<fr_grid(ctx->device, bound), FR_WARPS * 32, FR_SMEM, s>>>(t->level[l + 1], uniq, counts, (uint32_t)bound, t->level[l], refuse);
        ctx->stats.launches += 3;
        uint32_t* x = cur; cur = uniq; uniq = x; // the unique parents are the next level's (sorted) children
    }
    CU(cudaGetLastError());
    uint32_t refused = 0;
    CU(cudaMemcpyAsync(out_root, t->level[0], 32, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&refused, refuse, 4, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += 36;
    CU(cudaStreamSynchronize(s));
    return refused ? PHANT_GPU_E_INVALID : PHANT_GPU_OK; // refused: the trie is unchanged, out_root = its current root
}

extern "C" void phant_gpu_trie_close(phant_gpu_trie* t)
{
    if (!t) return;
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    t->store.release();
    t->work.release();
    t->leaf_rlp.release();
    if (t->sp) {
        SparseTrie* sp = t->sp;
        for (DevBuf* b : {&sp->rows[0], &sp->rows[1], &sp->arena, &sp->top, &sp->present, &sp->dirty, &sp->buckets, &sp->gather, &sp->gvals, &sp->sort})
            b->release();
        delete sp;
    }
    delete t;
}

// ------------------------------------------------------------------------------------------------
// Resident world state: the account trie (kind 1, above) and every account's storage trie, all on the device.  DESIGN.md §4.3c.
//
//   slot table   one sorted table for all accounts: rows (account key, slot key, 32-byte value), ordered by (account, slot)
//   account rows sorted by account key: storage root, slot count, storage depth L_a = st_target_L(n_a) (16..255 slots per
//                bucket, with the same hysteresis and premise fallback as kind 1) and the base of its dense top in a shared pool
//   pool         every account with L_a > 0 owns levels 0..L_a of 16-ary node references (32 B + presence byte per node)
//
// An apply sorts the diff, checks it, merges it into both tables, then rebuilds the dirty buckets of every touched account as
// ONE forest (build_forest with a per-segment start depth L_a) and re-hashes the dirty dense-top nodes of all accounts
// level by level (st_top_branch_kernel with per-node pool bases).  Accounts whose slot count crossed a depth bound, new and
// cleared accounts get all their buckets rebuilt in the same batch; accounts whose dense top lost a node down to one child are
// rebuilt one level lower in a further round.  The new storage roots feed account_fill_kernel, whose leaves go to the account
// trie without leaving the device.  Launches and read-backs depend on the largest L_a and the forest's depth, never on how
// many accounts an apply touches.
// ------------------------------------------------------------------------------------------------
namespace {

struct alignas(16) SlotRow { uint8_t akey[32], skey[32], val[32]; };
struct alignas(16) AccRow {
    uint8_t key[32], sroot[32];
    uint32_t n_slots, base;      // slots; first pool node of the dense top (valid for L_old)
    uint8_t L, L_old, full, pad; // storage depth (<= L_old once the region exists); depth the pool region was laid out for;
                                 // all buckets being rebuilt in the current round (the region does not hold a valid top yet)
    uint32_t pad2;
};
static_assert(sizeof(SlotRow) == 96 && sizeof(AccRow) == 80, "row layout");

// first slot row of account `akey` whose first L slot-key nibbles are >= want (want = 16^L: the account's end)
__device__ uint32_t slot_bucket_bound(const SlotRow* t, uint32_t n, const uint8_t* akey, uint32_t L, uint32_t want)
{
    uint32_t a = 0, b = n;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        const int c = cmp_key32(t[mid].akey, akey);
        if (c < 0 || (c == 0 && key_prefix(t[mid].skey, L) < want)) a = mid + 1; else b = mid;
    }
    return a;
}

// ---- staging of the diff ----
__global__ void rs_rank_kernel(const uint32_t* __restrict__ perm, uint32_t n, uint32_t* __restrict__ rank)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) rank[perm[i]] = i;
}
// listed accounts in key order: their rows as inserted, delete / clear flags, duplicate check
__global__ void rs_acc_dirty_kernel(const uint8_t* __restrict__ keys, const uint8_t* __restrict__ flags, const uint32_t* __restrict__ perm, uint32_t n,
                                    AccRow* __restrict__ rows, uint8_t* __restrict__ del, uint8_t* __restrict__ clear, uint32_t* __restrict__ counters)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t a = perm[i];
        AccRow r = {};
        for (int b = 0; b < 32; ++b) { r.key[b] = keys[32ull * a + b]; r.sroot[b] = EMPTY_ROOT_D[b]; }
        rows[i] = r;
        const uint8_t f = flags[a];
        del[i] = (f & PHANT_GPU_ACCOUNT_DELETE) ? 1 : 0;
        clear[i] = f ? 1 : 0; // DELETE or CLEAR_STORAGE: the account's existing slots go
        if (i + 1 < n && cmp_key32(keys + 32ull * a, keys + 32ull * perm[i + 1]) == 0) counters[0] = 1;
    }
}
// listed slots in (account, slot key) order: their rows, delete (zero value) / absent (account cleared) flags, duplicate check
__global__ void rs_slot_dirty_kernel(const uint8_t* __restrict__ akeys, const uint8_t* __restrict__ flags, const uint32_t* __restrict__ slot_acc,
                                     const uint8_t* __restrict__ skeys, const uint8_t* __restrict__ svals, const uint32_t* __restrict__ seg,
                                     const uint32_t* __restrict__ perm, uint32_t m, SlotRow* __restrict__ rows, uint32_t* __restrict__ acc_sorted,
                                     uint8_t* __restrict__ del, uint8_t* __restrict__ absent, uint32_t* __restrict__ counters)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint32_t q = perm[j], a = slot_acc[q];
        SlotRow r;
        uint32_t nz = 0;
        for (int b = 0; b < 32; ++b) { r.akey[b] = akeys[32ull * a + b]; r.skey[b] = skeys[32ull * q + b]; r.val[b] = svals[32ull * q + b]; nz |= r.val[b]; }
        rows[j] = r;
        acc_sorted[j] = seg[q];
        del[j] = nz ? 0 : 1;
        absent[j] = (flags[a] & PHANT_GPU_ACCOUNT_CLEAR_STORAGE) ? 1 : 0;
        if (j + 1 < m && seg[q] == seg[perm[j + 1]] && cmp_key32(skeys + 32ull * q, skeys + 32ull * perm[j + 1]) == 0) counters[1] = 1;
    }
}

// deleted and cleared accounts drop all their existing slots (warp per account); a deleted account that owned a dense top
// changes the pool layout
__global__ void rs_clear_slots_kernel(const SlotRow* __restrict__ S, uint32_t nS, const AccRow* __restrict__ A, const AccRow* __restrict__ rows,
                                      const uint8_t* __restrict__ clear, const uint8_t* __restrict__ akind, const uint32_t* __restrict__ alb, uint32_t na,
                                      uint32_t* __restrict__ del_flag, uint32_t* __restrict__ counters /*[2] slots dropped, [3] layout change*/)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < na; i += (gridDim.x * blockDim.x) >> 5) {
        if (!clear[i] || akind[i] == 0 || akind[i] == 2) continue; // absent before this apply: nothing to drop
        if (akind[i] == 3 && lane == 0 && A[alb[i]].L_old) counters[3] = 1;
        const uint32_t lo = slot_bucket_bound(S, nS, rows[i].key, 0, 0), hi = slot_bucket_bound(S, nS, rows[i].key, 0, 1);
        for (uint32_t r = lo + lane; r < hi; r += 32) del_flag[r] = 1;
        if (lane == 0) atomicAdd(&counters[2], hi - lo);
    }
}

// Upper bound of the dense-top nodes the listed accounts can own after this apply, from the pre-merge tables (read only):
// L_new <= max(L now, st_target_L(slots now + slots inserted)); counters64[0] += level_base(L_new + 1).  With every other
// region at most as large as it is laid out, the pool after this apply's one re-layout fits pool_nodes + this bound.
__global__ void rs_slot_ins_count_kernel(const uint32_t* __restrict__ sacc, const uint8_t* __restrict__ skind, uint32_t ms, uint32_t* __restrict__ ins)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < ms; j += gridDim.x * blockDim.x)
        if (skind[j] == 2) atomicAdd(&ins[sacc[j]], 1u);
}
__global__ void rs_pool_bound_kernel(const SlotRow* __restrict__ S, uint32_t nS, const AccRow* __restrict__ A, const AccRow* __restrict__ rows,
                                     const uint8_t* __restrict__ adel, const uint8_t* __restrict__ aclear, const uint8_t* __restrict__ akind,
                                     const uint32_t* __restrict__ alb, const uint32_t* __restrict__ ins, uint32_t na,
                                     unsigned long long* __restrict__ bound)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        if (adel[i]) continue;
        uint32_t n = ins[i], L = 0;
        if (akind[i] == 1 && !aclear[i]) {
            n += slot_bucket_bound(S, nS, rows[i].key, 0, 1) - slot_bucket_bound(S, nS, rows[i].key, 0, 0);
            L = A[alb[i]].L;
        }
        const uint32_t Lt = st_target_L(n);
        L = Lt > L ? Lt : L;
        if (L) atomicAdd(bound, (unsigned long long)level_base(L + 1));
    }
}

// ---- planning: which buckets of which account ----
struct Plan {
    uint32_t* row;   // listed account -> account row (NONE: deleted)
    uint32_t* dlo;   // its dirty slots [dlo, dhi) in sorted order
    uint32_t* dhi;
    uint8_t* L;      // its storage depth after this apply
    uint8_t* full;   // all buckets rebuilt
    uint8_t* active; // rebuilt in this round
    uint32_t* viol;  // its dense top broke the premise in this round
};
__global__ void rs_plan_kernel(AccRow* __restrict__ A, uint32_t nA, const SlotRow* __restrict__ S, uint32_t nS, const AccRow* __restrict__ rows,
                               const uint8_t* __restrict__ adel, const uint8_t* __restrict__ aclear, const uint8_t* __restrict__ akind,
                               const uint32_t* __restrict__ sacc, uint32_t ms, uint32_t na, uint32_t round, Plan p, uint32_t* __restrict__ counters)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        if (round) { // accounts whose dense top broke the premise: one level fewer, all buckets, inside the region they own
            p.active[i] = 0; // (levels 0..L-1 fit where levels 0..L were: only the first re-layout of an apply moves regions)
            if (!p.viol[i]) continue;
            AccRow& r = A[p.row[i]];
            r.L = (uint8_t)(r.L - 1);
            r.full = 1;
            p.L[i] = r.L;
            p.full[i] = 1;
            p.active[i] = 1;
            atomicMax(&counters[5], r.L);
            continue;
        }
        if (adel[i]) { p.row[i] = NONE; p.active[i] = 0; continue; }
        const uint8_t* key = rows[i].key;
        const uint32_t ri = row_lower_bound<AccRow, 32>(A, nA, key);
        AccRow& r = A[ri];
        const uint32_t n = slot_bucket_bound(S, nS, key, 0, 1) - slot_bucket_bound(S, nS, key, 0, 0);
        const uint32_t Lt = st_target_L(n);
        const bool full = akind[i] == 2 || aclear[i] || Lt > r.L || Lt + 1 < r.L;
        const uint32_t L = full ? Lt : r.L;
        uint32_t a = 0, b = ms; // dirty slots of listed account i (sorted by account)
        while (a < b) { const uint32_t mid = (a + b) >> 1; if (sacc[mid] < i) a = mid + 1; else b = mid; }
        uint32_t c = a, d = ms;
        while (c < d) { const uint32_t mid = (c + d) >> 1; if (sacc[mid] < i + 1) c = mid + 1; else d = mid; }
        r.n_slots = n;
        r.L = (uint8_t)L;
        r.full = full ? 1 : 0;
        if (L != r.L_old) counters[3] = 1; // the pool layout changes (L_old == L == 0 never gets here)
        p.row[i] = ri; p.dlo[i] = a; p.dhi[i] = c; p.L[i] = (uint8_t)L; p.full[i] = full ? 1 : 0;
        p.active[i] = full || c > a;
        if (p.active[i]) atomicMax(&counters[5], L);
    }
}
// first dirty slot of each dirty bucket of the accounts rebuilt incrementally
__global__ void rs_slot_first_kernel(const SlotRow* __restrict__ dirty, const uint32_t* __restrict__ sacc, uint32_t ms, Plan p, uint32_t* __restrict__ first)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j <= ms; j += gridDim.x * blockDim.x) {
        if (j == ms) { first[j] = 0; break; }
        const uint32_t i = sacc[j];
        const uint32_t L = p.L[i];
        first[j] = p.active[i] && !p.full[i] &&
                   (j == p.dlo[i] || key_prefix(dirty[j].skey, L) != key_prefix(dirty[j - 1].skey, L));
    }
}
__global__ void rs_bucket_count_kernel(const uint32_t* __restrict__ F, uint32_t na, Plan p, uint32_t* __restrict__ cnt)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= na; i += gridDim.x * blockDim.x)
        cnt[i] = i == na || !p.active[i] ? 0 : (p.full[i] ? 1u << (4 * p.L[i]) : F[p.dhi[i]] - F[p.dlo[i]]);
}
// the work list: (listed account, bucket) pairs, sorted by account then bucket
__global__ void rs_fill_entries_kernel(const SlotRow* __restrict__ dirty, const uint32_t* __restrict__ sacc, uint32_t ms, const uint32_t* __restrict__ first,
                                       const uint32_t* __restrict__ F, const uint32_t* __restrict__ off, uint32_t na, Plan p,
                                       uint32_t* __restrict__ e_acc, uint32_t* __restrict__ e_b)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < ms; j += gridDim.x * blockDim.x)
        if (first[j]) {
            const uint32_t i = sacc[j], e = off[i] + F[j] - F[p.dlo[i]];
            e_acc[e] = i;
            e_b[e] = key_prefix(dirty[j].skey, p.L[i]);
        }
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < na; i += (gridDim.x * blockDim.x) >> 5)
        if (p.active[i] && p.full[i])
            for (uint32_t b = lane; b < (1u << (4 * p.L[i])); b += 32) { e_acc[off[i] + b] = i; e_b[off[i] + b] = b; }
}
__global__ void rs_entry_range_kernel(const SlotRow* __restrict__ S, uint32_t nS, const AccRow* __restrict__ A, const uint32_t* __restrict__ e_acc,
                                      const uint32_t* __restrict__ e_b, uint32_t E, Plan p, uint32_t* __restrict__ lo, uint32_t* __restrict__ cnt,
                                      uint32_t* __restrict__ start)
{
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e <= E; e += gridDim.x * blockDim.x) {
        if (e == E) { cnt[e] = 0; break; }
        const uint32_t i = e_acc[e], L = p.L[i];
        const uint8_t* key = A[p.row[i]].key;
        const uint32_t a = slot_bucket_bound(S, nS, key, L, e_b[e]), b = slot_bucket_bound(S, nS, key, L, e_b[e] + 1);
        lo[e] = a;
        cnt[e] = b - a;
        start[e] = L;
    }
}
// forest input: row index (in 32-byte units of the slot table, see storage_fill_kernel) and segment of every key (warp per bucket)
__global__ void rs_gather_kernel(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ seg_off, uint32_t E, uint32_t* __restrict__ unit,
                                 uint32_t* __restrict__ seg_of_key)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < E; e += (gridDim.x * blockDim.x) >> 5)
        for (uint32_t t = seg_off[e] + lane; t < seg_off[e + 1]; t += 32) {
            unit[t] = 3 * (lo[e] + t - seg_off[e]);
            seg_of_key[t] = e;
        }
}
__global__ void rs_scatter_roots_kernel(const uint8_t* __restrict__ roots, const uint32_t* __restrict__ e_acc, const uint32_t* __restrict__ e_b,
                                        const uint32_t* __restrict__ cnt, uint32_t E, Plan p, AccRow* __restrict__ A, uint8_t* __restrict__ top,
                                        uint8_t* __restrict__ present)
{
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
        const uint32_t i = e_acc[e], L = p.L[i];
        AccRow& r = A[p.row[i]];
        uint8_t* dst = r.sroot; // L == 0: the bucket is the whole storage trie
        if (L) {
            const uint64_t node = r.base + level_base(L) + e_b[e];
            dst = top + 32 * node;
            present[node] = cnt[e] ? 1 : 0;
        }
        for (int b = 0; b < 32; ++b) dst[b] = roots[32ull * e + b];
    }
}
// dense-top nodes of depth d above the entries: flags of the first entry of each distinct node
__global__ void rs_node_flag_kernel(const uint32_t* __restrict__ e_acc, const uint32_t* __restrict__ e_b, uint32_t E, uint32_t d, Plan p,
                                    uint32_t* __restrict__ first)
{
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e <= E; e += gridDim.x * blockDim.x) {
        if (e == E) { first[e] = 0; break; }
        const uint32_t i = e_acc[e], L = p.L[i];
        first[e] = L > d && (e == 0 || e_acc[e - 1] != i || (e_b[e - 1] >> (4 * (L - d))) != (e_b[e] >> (4 * (L - d))));
    }
}
__global__ void rs_node_list_kernel(const uint32_t* __restrict__ e_acc, const uint32_t* __restrict__ e_b, const uint32_t* __restrict__ first,
                                    const uint32_t* __restrict__ pos, uint32_t E, uint32_t d, Plan p, const AccRow* __restrict__ A,
                                    uint32_t* __restrict__ par, uint32_t* __restrict__ base, uint32_t* __restrict__ owner)
{
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x)
        if (first[e]) {
            const uint32_t i = e_acc[e];
            par[pos[e]] = e_b[e] >> (4 * (p.L[i] - d));
            base[pos[e]] = A[p.row[i]].base;
            owner[pos[e]] = i;
        }
}
// end of a round: the storage roots of its accounts with a dense top, and their regions marked valid again (a later
// re-layout copies them)
__global__ void rs_top_root_kernel(uint32_t na, Plan p, AccRow* __restrict__ A, const uint8_t* __restrict__ top, const uint8_t* __restrict__ present)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        if (!p.active[i]) continue;
        AccRow& r = A[p.row[i]];
        r.full = 0;
        if (!p.L[i]) continue;
        const uint8_t* src = present[r.base] ? top + 32ull * r.base : EMPTY_ROOT_D;
        for (int b = 0; b < 32; ++b) r.sroot[b] = src[b];
    }
}
// pool layout: every account row with L > 0 gets level_base(L + 1) nodes; regions still valid move along
__global__ void rs_pool_size_kernel(const AccRow* __restrict__ A, uint32_t nA, uint64_t* __restrict__ size)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < nA; r += gridDim.x * blockDim.x) size[r] = A[r].L ? level_base(A[r].L + 1) : 0;
}
__global__ void rs_pool_move_kernel(AccRow* __restrict__ A, uint32_t nA, const uint64_t* __restrict__ nbase, const uint8_t* __restrict__ old_top,
                                    const uint8_t* __restrict__ old_present, uint8_t* __restrict__ top, uint8_t* __restrict__ present)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nA; r += (gridDim.x * blockDim.x) >> 5) {
        AccRow& a = A[r];
        if (a.L && a.L <= a.L_old && !a.full) { // a valid top of depth L (possibly lowered inside a larger region)
            const uint64_t from = a.base, to = nbase[r], total = level_base(a.L + 1);
            const uint4* s = reinterpret_cast<const uint4*>(old_top + 32 * from);
            uint4* t = reinterpret_cast<uint4*>(top + 32 * to);
            for (uint64_t k = lane; k < 2 * total; k += 32) t[k] = s[k];
            for (uint64_t k = lane; k < total; k += 32) present[to + k] = old_present[from + k];
        }
        __syncwarp();
        if (lane == 0) { a.base = (uint32_t)nbase[r]; a.L_old = a.L; }
    }
}
// storage roots out (caller's order, zero for deleted accounts); the apply's marks cleared
__global__ void rs_roots_out_kernel(const uint32_t* __restrict__ perm, uint32_t na, Plan p, AccRow* __restrict__ A, uint8_t* __restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        uint8_t* o = out + 32ull * perm[i];
        if (p.row[i] == NONE) { for (int b = 0; b < 32; ++b) o[b] = 0; continue; }
        AccRow& r = A[p.row[i]];
        for (int b = 0; b < 32; ++b) o[b] = r.sroot[b];
    }
}
// account-trie values: upserted accounts' leaves at avo[0..n_up], deleted accounts after them with empty values
__global__ void rs_acc_voff_kernel(const uint64_t* __restrict__ avo, uint32_t n_up, uint32_t na, uint32_t* __restrict__ voff)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= na; i += gridDim.x * blockDim.x) voff[i] = (uint32_t)avo[i < n_up ? i : n_up];
}

} // namespace
// P's account-body decoder, for the old account of an undo record, the per-key reads of the state (resident_read.cuh), and the
// node decoder (transition.cuh) and chain walks over a node set (proof_chain.cuh) of T, the proofs and the trie nodes.  Their
// headers open an anonymous namespace inside `phant`; wrapped in a namespace of their own so that they do not meet this file's
// anonymous namespace through `using namespace phant`.
namespace rs_body {
#include "state_read.cuh"
#include "resident_read.cuh"
#include "resident_range.cuh"
#include "snap_range.cuh"
#include "proof_chain.cuh"
}
namespace tn = rs_body::phant;
using rs_body::phant::AccountBody;
using rs_body::phant::decode_account_body;
using rs_body::phant::listed_slots;
namespace {

// ---- undo records (phant_gpu_resident_state_set_journal): the inverse of an apply, captured from the pre-merge tables ----
// the account body a present listed account has now, from the account trie's leaf (its row table holds the same sorted key
// set as the account rows, so the row's lower bound indexes it)
__device__ __forceinline__ bool old_account(const KRow* krows, const uint8_t* arena, uint32_t r, const uint8_t* key, AccountBody& b, const uint8_t*& body)
{
    if (cmp_key32(krows[r].key, key) != 0) return false;
    body = arena + krows[r].off;
    return decode_account_body(body, krows[r].len, b);
}
// per listed account: whether the record lists it, and how many slots the record holds for it
__global__ void rs_undo_size_kernel(const AccRow* __restrict__ rows, const uint8_t* __restrict__ aclear, const uint8_t* __restrict__ akind,
                                    const uint32_t* __restrict__ alb, uint32_t na, const SlotRow* __restrict__ S, uint32_t nS,
                                    const uint32_t* __restrict__ sacc, uint32_t ms, const KRow* __restrict__ krows,
                                    const uint8_t* __restrict__ arena, uint32_t* __restrict__ listed, uint32_t* __restrict__ nslots,
                                    uint32_t* __restrict__ bad)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= na; i += gridDim.x * blockDim.x) {
        if (i == na) { listed[i] = 0; nslots[i] = 0; break; }
        const uint8_t k = akind[i];
        listed[i] = k != 0; // absent and deleted: nothing to undo
        nslots[i] = 0;
        if (k == 0 || k == 2) continue; // absent and upserted: the record deletes it
        AccountBody b;
        const uint8_t* body;
        if (!old_account(krows, arena, alb[i], rows[i].key, b, body)) *bad = 1;
        uint32_t lo, hi;
        if (aclear[i]) { lo = slot_bucket_bound(S, nS, rows[i].key, 0, 0); hi = slot_bucket_bound(S, nS, rows[i].key, 0, 1); }
        else listed_slots(sacc, ms, i, lo, hi);
        nslots[i] = hi - lo;
    }
}
// the record, in the layout of a staged diff (warp per listed account): a present account gets its old nonce, balance and
// codeHash, with CLEAR_STORAGE and every slot it held when the apply drops its storage, else the old value of every listed slot
// (zero where the slot was absent); an absent upserted account gets DELETE
__global__ void rs_undo_fill_kernel(const AccRow* __restrict__ rows, const uint8_t* __restrict__ aclear, const uint8_t* __restrict__ akind,
                                    const uint32_t* __restrict__ alb, uint32_t na, const SlotRow* __restrict__ S, uint32_t nS,
                                    const SlotRow* __restrict__ srows, const uint32_t* __restrict__ sacc, const uint8_t* __restrict__ skind,
                                    const uint32_t* __restrict__ slb, uint32_t ms, const KRow* __restrict__ krows,
                                    const uint8_t* __restrict__ arena, const uint32_t* __restrict__ apos,
                                    const uint32_t* __restrict__ soff, uint8_t* __restrict__ akeys, uint8_t* __restrict__ aflags,
                                    uint64_t* __restrict__ nonce, uint8_t* __restrict__ bal, uint8_t* __restrict__ code,
                                    uint32_t* __restrict__ racc, uint8_t* __restrict__ skeys, uint8_t* __restrict__ svals)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < na; i += (gridDim.x * blockDim.x) >> 5) {
        const uint8_t k = akind[i];
        if (k == 0) continue;
        const uint32_t p = apos[i], o = soff[i];
        const uint8_t* key = rows[i].key;
        akeys[32ull * p + lane] = key[lane];
        if (k == 2) {
            bal[32ull * p + lane] = 0;
            code[32ull * p + lane] = 0;
            if (lane == 0) { aflags[p] = PHANT_GPU_ACCOUNT_DELETE; nonce[p] = 0; }
            continue;
        }
        AccountBody b;
        const uint8_t* body;
        old_account(krows, arena, alb[i], key, b, body); // checked by rs_undo_size_kernel
        bal[32ull * p + lane] = lane < 32 - b.bal_len ? 0 : body[b.bal_off + lane - (32 - b.bal_len)];
        code[32ull * p + lane] = body[b.code_off + lane];
        if (lane == 0) { aflags[p] = aclear[i] ? PHANT_GPU_ACCOUNT_CLEAR_STORAGE : 0; nonce[p] = b.nonce; }
        if (aclear[i]) {
            const uint32_t lo = slot_bucket_bound(S, nS, key, 0, 0), hi = slot_bucket_bound(S, nS, key, 0, 1);
            for (uint32_t r = lo + lane; r < hi; r += 32) {
                const uint64_t q = o + r - lo;
                const uint4* src = reinterpret_cast<const uint4*>(S + r);
                uint4* k4 = reinterpret_cast<uint4*>(skeys + 32 * q);
                uint4* v4 = reinterpret_cast<uint4*>(svals + 32 * q);
                k4[0] = src[2]; k4[1] = src[3]; v4[0] = src[4]; v4[1] = src[5];
                racc[q] = p;
            }
        } else {
            uint32_t lo, hi;
            listed_slots(sacc, ms, i, lo, hi);
            for (uint32_t j = lo + lane; j < hi; j += 32) {
                const uint64_t q = o + j - lo;
                const uint4* src = reinterpret_cast<const uint4*>(srows + j);
                uint4* k4 = reinterpret_cast<uint4*>(skeys + 32 * q);
                uint4* v4 = reinterpret_cast<uint4*>(svals + 32 * q);
                k4[0] = src[2]; k4[1] = src[3];
                if (skind[j] == 1 || skind[j] == 3) { // the slot existed: its old value
                    const uint4* old = reinterpret_cast<const uint4*>(S + slb[j]);
                    v4[0] = old[4]; v4[1] = old[5];
                } else v4[0] = v4[1] = make_uint4(0, 0, 0, 0);
                racc[q] = p;
            }
        }
    }
}
// the record's old storage roots, for reads at past roots (revert does not replay them): a present account's from its old
// body, zero for a DELETE account
__global__ void rs_undo_sroot_kernel(const AccRow* __restrict__ rows, const uint8_t* __restrict__ akind, const uint32_t* __restrict__ alb,
                                     uint32_t na, const KRow* __restrict__ krows, const uint8_t* __restrict__ arena,
                                     const uint32_t* __restrict__ apos, uint8_t* __restrict__ sroot)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        const uint8_t k = akind[i];
        if (k == 0) continue;
        uint8_t* d = sroot + 32ull * apos[i];
        AccountBody b;
        const uint8_t* body;
        if (k == 2 || !old_account(krows, arena, alb[i], rows[i].key, b, body)) { // (decoding checked by rs_undo_size_kernel)
            for (int j = 0; j < 32; ++j) d[j] = 0;
            continue;
        }
        for (int j = 0; j < 32; ++j) d[j] = body[b.root_off + j];
    }
}
// upserted / deleted accounts in the caller's order, for a diff that exists only on the device (a replayed record)
__global__ void rs_up_flag_kernel(const uint8_t* __restrict__ aflags, uint32_t na, uint32_t* __restrict__ up)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= na; i += gridDim.x * blockDim.x)
        up[i] = i < na && !(aflags[i] & PHANT_GPU_ACCOUNT_DELETE);
}
__global__ void rs_partition_kernel(const uint32_t* __restrict__ up, const uint32_t* __restrict__ pos, uint32_t na, uint32_t* __restrict__ idx)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x)
        idx[up[i] ? pos[i] : pos[na] + i - pos[i]] = i;
}

// ---- witnesses (phant_gpu_resident_state_witness): the pre-state paths of the proof keys, nothing resident written ----
// Trie 0 is the account trie, trie 1 + i the storage trie of listed account i (key order).  ok: the witness proves keys in it
// (for a storage trie: the account is present, neither deleted nor cleared, and has slots); L and base: its dense top;
// [slo, shi): its rows in the slot table.
struct WitTries { uint8_t* ok; uint32_t *L, *base, *slo, *shi; };
struct WitTops { const uint8_t *acc_top, *acc_present, *pool_top, *pool_present; };
__global__ void wit_tries_kernel(const AccRow* __restrict__ A, const SlotRow* __restrict__ S, uint32_t nS, const AccRow* __restrict__ rows,
                                 const uint8_t* __restrict__ aclear, const uint8_t* __restrict__ akind, const uint32_t* __restrict__ alb, uint32_t na,
                                 uint32_t acc_n, uint32_t acc_L, WitTries w)
{
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t <= na; t += gridDim.x * blockDim.x) {
        if (t == 0) { w.ok[0] = acc_n != 0; w.L[0] = acc_L; w.base[0] = 0; w.slo[0] = w.shi[0] = 0; continue; }
        const uint32_t i = t - 1;
        const uint32_t lo = slot_bucket_bound(S, nS, rows[i].key, 0, 0), hi = slot_bucket_bound(S, nS, rows[i].key, 0, 1);
        const bool ok = akind[i] == 1 && !aclear[i] && hi > lo;
        w.ok[t] = ok;
        w.L[t] = ok ? A[alb[i]].L : 0;
        w.base[t] = ok ? A[alb[i]].base : 0;
        w.slo[t] = lo;
        w.shi[t] = hi;
    }
}
__device__ __forceinline__ void wit_put(uint8_t* ckeys, uint32_t* cseg, uint32_t c, const uint8_t* key, uint32_t trie)
{
    for (int b = 0; b < 32; ++b) ckeys[32ull * c + b] = key[b];
    cseg[c] = trie;
}
// whether the diff deletes account `key` (the listed rows are sorted)
__device__ bool wit_acc_gone(const AccRow* rows, const uint8_t* adel, uint32_t na, const uint8_t* key)
{
    const uint32_t a = row_lower_bound<AccRow, 32>(rows, na, key);
    return a < na && adel[a] && cmp_key32(rows[a].key, key) == 0;
}
// proof-key candidates 3i .. 3i+2 of listed account i: its key, and for a deleted one the nearest account keys before and
// after it that the diff does not delete (cseg NONE: no candidate).  Each neighbour walk steps over the table keys the diff
// also deletes, one binary search per step: a run of k adjacent deleted keys costs O(k log k) per thread and O(k^2 log k)
// in all.  A block deletes at most a few thousand accounts, so the runs stay short; a diff that deletes most of a large
// state pays for it here (wit_slot_keys_kernel is the same for zeroed slots).
__global__ void wit_acc_keys_kernel(const AccRow* __restrict__ rows, const uint8_t* __restrict__ adel, uint32_t na, const KRow* __restrict__ krows,
                                    uint32_t n, uint8_t* __restrict__ ckeys, uint32_t* __restrict__ cseg, uint32_t* __restrict__ count)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        const uint32_t c = 3 * i;
        cseg[c] = cseg[c + 1] = cseg[c + 2] = NONE;
        if (n == 0) continue;
        const uint8_t* key = rows[i].key;
        wit_put(ckeys, cseg, c, key, 0);
        uint32_t got = 1;
        if (adel[i]) {
            const uint32_t lb = row_lower_bound<KRow, 32>(krows, n, key);
            int64_t j = (int64_t)lb - 1;
            while (j >= 0 && wit_acc_gone(rows, adel, na, krows[j].key)) --j;
            if (j >= 0) { wit_put(ckeys, cseg, c + 1, krows[j].key, 0); ++got; }
            uint32_t q = lb + (lb < n && cmp_key32(krows[lb].key, key) == 0 ? 1 : 0);
            while (q < n && wit_acc_gone(rows, adel, na, krows[q].key)) ++q;
            if (q < n) { wit_put(ckeys, cseg, c + 2, krows[q].key, 0); ++got; }
        }
        atomicAdd(count, got);
    }
}
// candidates c0 + 3j .. c0 + 3j+2 of listed slot j (sorted order): its key in its account's storage trie, and for a zero write
// the nearest slot keys of that account before and after it that the diff does not zero
__global__ void wit_slot_keys_kernel(const SlotRow* __restrict__ srows, const uint32_t* __restrict__ sacc, const uint8_t* __restrict__ sdel,
                                     uint32_t ms, const SlotRow* __restrict__ S, uint32_t nS, WitTries w, uint32_t c0, uint8_t* __restrict__ ckeys,
                                     uint32_t* __restrict__ cseg, uint32_t* __restrict__ count)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < ms; j += gridDim.x * blockDim.x) {
        const uint32_t c = c0 + 3 * j, i = sacc[j], t = i + 1;
        cseg[c] = cseg[c + 1] = cseg[c + 2] = NONE;
        if (!w.ok[t]) continue;
        wit_put(ckeys, cseg, c, srows[j].skey, t);
        uint32_t got = 1;
        if (sdel[j]) {
            uint32_t dlo, dhi;
            listed_slots(sacc, ms, i, dlo, dhi);
            auto gone = [&](const uint8_t* skey) { // the diff zeroes this slot of account i
                uint32_t a = dlo, b = dhi;
                while (a < b) { const uint32_t mid = (a + b) >> 1; if (cmp_key32(srows[mid].skey, skey) < 0) a = mid + 1; else b = mid; }
                return a < dhi && sdel[a] && cmp_key32(srows[a].skey, skey) == 0;
            };
            const uint32_t lo = w.slo[t], hi = w.shi[t], lb = row_lower_bound<SlotRow, 64>(S, nS, srows[j].akey);
            int64_t r = (int64_t)lb - 1;
            while (r >= (int64_t)lo && gone(S[r].skey)) --r;
            if (r >= (int64_t)lo) { wit_put(ckeys, cseg, c + 1, S[r].skey, t); ++got; }
            uint32_t q = lb + (lb < hi && cmp_key32(S[lb].skey, srows[j].skey) == 0 ? 1 : 0);
            while (q < hi && gone(S[q].skey)) ++q;
            if (q < hi) { wit_put(ckeys, cseg, c + 2, S[q].skey, t); ++got; }
        }
        atomicAdd(count, got);
    }
}
__global__ void wit_proof_keys_kernel(const uint8_t* __restrict__ ckeys, const uint32_t* __restrict__ cseg, const uint32_t* __restrict__ perm,
                                      uint32_t np, uint8_t* __restrict__ pkeys, uint32_t* __restrict__ ptrie)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < np; j += gridDim.x * blockDim.x) {
        const uint32_t c = perm[j];
        const uint4* s = reinterpret_cast<const uint4*>(ckeys + 32ull * c);
        uint4* d = reinterpret_cast<uint4*>(pkeys + 32ull * j);
        d[0] = s[0]; d[1] = s[1];
        ptrie[j] = cseg[c];
    }
}
// The dense-top nodes on the proof keys' paths, each encoded once (by the first proof key of its trie below it) from its 16
// child references, as st_top_branch_kernel encodes it; its digest is the reference its parent holds.  Every node of a dense
// top has two children or more, each a 32-byte hash.
__global__ void wit_dense_kernel(const uint8_t* __restrict__ pkeys, const uint32_t* __restrict__ ptrie, uint32_t np, WitTries w, WitTops tp,
                                 WitnessOut out)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < np; j += gridDim.x * blockDim.x) {
        const uint32_t t = ptrie[j], L = w.L[t];
        const uint64_t base = w.base[t];
        const uint8_t* top = t ? tp.pool_top : tp.acc_top;
        const uint8_t* present = t ? tp.pool_present : tp.acc_present;
        const uint8_t* key = pkeys + 32ull * j;
        for (uint32_t d = 0; d < L; ++d) {
            const uint32_t idx = key_prefix(key, d);
            if (j && ptrie[j - 1] == t && key_prefix(key - 32, d) == idx) continue;
            const uint64_t node = base + level_base(d) + idx, c0 = base + level_base(d + 1) + 16ull * idx;
            if (!present[node]) break; // the key's path leaves the trie above this level
            uint32_t mask = 0;
            for (uint32_t v = 0; v < 16; ++v) mask |= (present[c0 + v] ? 1u : 0u) << v;
            const uint32_t c = __popc(mask), payload = 33 * c + (16 - c) + 1;
            const uint32_t hdr = payload <= 55 ? 1 : payload < 256 ? 2 : 3;
            uint8_t* o = wit_reserve(out, hdr + payload, top + 32 * node);
            if (!o) continue;
            if (hdr == 1) *o++ = (uint8_t)(0xc0 + payload);
            else if (hdr == 2) { *o++ = 0xf8; *o++ = (uint8_t)payload; }
            else { *o++ = 0xf9; *o++ = (uint8_t)(payload >> 8); *o++ = (uint8_t)payload; }
            for (uint32_t v = 0; v < 16; ++v) {
                if (!((mask >> v) & 1)) { *o++ = 0x80; continue; }
                *o++ = 0xa0;
                for (int b = 0; b < 32; ++b) *o++ = top[32 * (c0 + v) + b];
            }
            *o = 0x80;
        }
    }
}
// first proof key of each (trie, bucket) whose bucket holds keys
__global__ void wit_bucket_flag_kernel(const uint8_t* __restrict__ pkeys, const uint32_t* __restrict__ ptrie, uint32_t np, WitTries w, WitTops tp,
                                       uint32_t* __restrict__ first)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j <= np; j += gridDim.x * blockDim.x) {
        if (j == np) { first[j] = 0; continue; }
        const uint32_t t = ptrie[j], L = w.L[t], b = key_prefix(pkeys + 32ull * j, L);
        bool f = !(j && ptrie[j - 1] == t && key_prefix(pkeys + 32ull * (j - 1), L) == b);
        if (f && L) f = (t ? tp.pool_present : tp.acc_present)[w.base[t] + level_base(L) + b] != 0;
        first[j] = f;
    }
}
__device__ uint32_t krow_bucket_bound(const KRow* t, uint32_t n, uint32_t L, uint32_t want)
{
    if (!L) return want ? n : 0;
    uint32_t a = 0, b = n;
    while (a < b) { const uint32_t mid = (a + b) >> 1; if (key_prefix(t[mid].key, L) < want) a = mid + 1; else b = mid; }
    return a;
}
// the buckets to rebuild: trie, start depth and table range of each (ecnt[E] = 0 for the scan)
__global__ void wit_bucket_kernel(const uint8_t* __restrict__ pkeys, const uint32_t* __restrict__ ptrie, uint32_t np, const uint32_t* __restrict__ first,
                                  const uint32_t* __restrict__ pos, WitTries w, const KRow* __restrict__ krows, uint32_t n, const SlotRow* __restrict__ S,
                                  uint32_t nS, const AccRow* __restrict__ rows, uint32_t* __restrict__ etrie, uint32_t* __restrict__ elo,
                                  uint32_t* __restrict__ ecnt, uint32_t* __restrict__ estart)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j <= np; j += gridDim.x * blockDim.x) {
        if (j == np) { ecnt[pos[np]] = 0; continue; }
        if (!first[j]) continue;
        const uint32_t e = pos[j], t = ptrie[j], L = w.L[t], b = key_prefix(pkeys + 32ull * j, L);
        uint32_t lo, hi;
        if (t == 0) { lo = krow_bucket_bound(krows, n, L, b); hi = krow_bucket_bound(krows, n, L, b + 1); }
        else { lo = slot_bucket_bound(S, nS, rows[t - 1].key, L, b); hi = slot_bucket_bound(S, nS, rows[t - 1].key, L, b + 1); }
        etrie[e] = t; elo[e] = lo; ecnt[e] = hi - lo; estart[e] = L;
    }
}
__device__ __forceinline__ uint32_t slot_value_size(const uint8_t* v)
{
    uint32_t z = 0;
    while (z < 32 && v[z] == 0) ++z;
    return (32 - z == 1 && v[z] < 0x80) ? 1 : 1 + (32 - z);
}
// forest input of the buckets (warp per bucket): keys, segment of each key, its table row and value size
__global__ void wit_forest_keys_kernel(const uint32_t* __restrict__ etrie, const uint32_t* __restrict__ elo, const uint32_t* __restrict__ seg_off,
                                       uint32_t E, uint32_t mk, const KRow* __restrict__ krows, const SlotRow* __restrict__ S, uint8_t* __restrict__ fk,
                                       uint32_t* __restrict__ fko, uint32_t* __restrict__ seg_of_key, uint32_t* __restrict__ src, uint64_t* __restrict__ vsize)
{
    const uint32_t lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0) fko[mk] = 32u * mk;
    for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < E; e += (gridDim.x * blockDim.x) >> 5)
        for (uint32_t q = seg_off[e] + lane; q < seg_off[e + 1]; q += 32) {
            const uint32_t row = elo[e] + q - seg_off[e];
            const uint8_t* key = etrie[e] ? S[row].skey : krows[row].key;
            const uint4* s = reinterpret_cast<const uint4*>(key);
            uint4* d = reinterpret_cast<uint4*>(fk + 32ull * q);
            d[0] = s[0]; d[1] = s[1];
            fko[q] = 32u * q;
            seg_of_key[q] = e;
            src[q] = row;
            vsize[q] = etrie[e] ? slot_value_size(S[row].val) : krows[row].len;
        }
}
// leaf values: the account trie's from its arena, a slot's as rlp(value without leading zeros)
__global__ void wit_forest_vals_kernel(const uint32_t* __restrict__ etrie, const uint32_t* __restrict__ seg_of_key, const uint32_t* __restrict__ src,
                                       const uint64_t* __restrict__ voff, uint32_t mk, const KRow* __restrict__ krows, const uint8_t* __restrict__ arena,
                                       const SlotRow* __restrict__ S, uint8_t* __restrict__ fv)
{
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < mk; q += gridDim.x * blockDim.x) {
        const uint32_t row = src[q];
        uint8_t* o = fv + voff[q];
        if (etrie[seg_of_key[q]] == 0) {
            const uint8_t* v = arena + krows[row].off;
            for (uint32_t b = 0; b < krows[row].len; ++b) o[b] = v[b];
            continue;
        }
        const uint8_t* v = S[row].val;
        uint32_t z = 0;
        while (z < 32 && v[z] == 0) ++z;
        if (!(32 - z == 1 && v[z] < 0x80)) *o++ = (uint8_t)(0x80 + 32 - z);
        for (uint32_t b = z; b < 32; ++b) *o++ = v[b];
    }
}
// exported nodes sorted by digest: the first of each digest is kept
__global__ void wit_unique_kernel(const uint8_t* __restrict__ digests, const WNode* __restrict__ nodes, const uint32_t* __restrict__ perm, uint32_t n,
                                  uint32_t* __restrict__ keep, uint64_t* __restrict__ size)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j <= n; j += gridDim.x * blockDim.x) {
        if (j == n) { keep[j] = 0; size[j] = 0; continue; }
        const uint32_t p = perm[j];
        bool k = j == 0;
        if (!k) {
            const uint8_t *a = digests + 32ull * p, *b = digests + 32ull * perm[j - 1];
            for (int q = 0; q < 32 && !k; ++q) k = a[q] != b[q];
        }
        keep[j] = k;
        size[j] = k ? nodes[p].len : 0;
    }
}
// the CSR (warp per node): node_off first, then the bytes
__global__ void wit_write_kernel(const uint8_t* __restrict__ bytes, const WNode* __restrict__ nodes, const uint32_t* __restrict__ perm,
                                 const uint32_t* __restrict__ keep, const uint32_t* __restrict__ idx, const uint64_t* __restrict__ offs, uint32_t n,
                                 uint64_t* __restrict__ node_off, uint8_t* __restrict__ out)
{
    const uint32_t lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0) node_off[idx[n]] = offs[n];
    for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += (gridDim.x * blockDim.x) >> 5) {
        if (!keep[j]) continue;
        const WNode w = nodes[perm[j]];
        if (lane == 0) node_off[idx[j]] = offs[j];
        for (uint32_t b = lane; b < w.len; b += 32) out[offs[j] + b] = bytes[w.off + b];
    }
}
// the kept nodes' digests in the CSR's order, for the proofs' chain walk
__global__ void prf_digest_kernel(const uint8_t* __restrict__ digests, const uint32_t* __restrict__ perm, const uint32_t* __restrict__ keep,
                                  const uint32_t* __restrict__ idx, uint32_t n, uint8_t* __restrict__ out)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        if (!keep[j]) continue;
        const uint4* s = reinterpret_cast<const uint4*>(digests + 32ull * perm[j]);
        uint4* d = reinterpret_cast<uint4*>(out + 32ull * idx[j]);
        d[0] = s[0]; d[1] = s[1];
    }
}

} // namespace

struct phant_gpu_resident_state {
    phant_gpu_ctx* ctx;
    SparseTrie acct_sp;         // kind 1's table: account key -> rlp([nonce, balance, storageRoot, codeHash])
    DevBuf S[2], A[2], pool[2]; // slot table, account rows, dense-top pool (32-byte references, then presence bytes)
    int sc = 0, ac = 0, pc = 0;
    uint32_t nS = 0, nA = 0;
    uint64_t pool_nodes = 0;
    DevBuf in, dirty, work, forest, sort; // scratch
    bool writing = false; // the current apply has started to change resident data
    bool failed = false;  // an apply failed after its first write: the tables may disagree, every later call is refused
    // undo journal: one record per successful apply, newest last; a record is a diff on the device (the staging layout) that
    // takes the state back to `root`, followed by its accounts' old storage roots (for reads at past roots)
    struct Record { DevBuf buf; uint32_t na = 0, ms = 0; uint8_t root[32]; };
    uint32_t depth = 0;
    std::deque<Record> journal;
    Record next;               // the record the current apply captures into
    std::vector<DevBuf> spare; // buffers of dropped and undone records, reused
    // the one result a witness, prove, trie_nodes or snap_ranges call holds until its copy call or another call comes (`held`:
    // its kind): the node set as CSR in wit_res (scratch for trie nodes), the proofs' chains and values in prf_res, the trie
    // nodes' status, node offsets and served bytes in tnd_res (DESIGN.md §4.3k), the snap answers' entries, bodies and proof
    // lists in snp_res (§4.3m); wit_out holds the exported nodes (scratch)
    enum class Result { NONE, WITNESS, PROOFS, TRIE_NODES, SNAP_RANGES };
    Result held = Result::NONE;
    DevBuf wit_out, wit_res, prf_res, tnd_res, snp_res;
    uint64_t wit_n = 0, wit_bytes = 0;
    uint32_t prf_na = 0, prf_ms = 0; // the proofs held: accounts, slots, chain entries
    uint64_t prf_refs = 0;
    uint32_t tnd_n = 0;             // the trie nodes held: paths, paths served, their bytes
    uint64_t tnd_nodes = 0, tnd_bytes = 0;
    // the snap answers held: requests of each kind, then the sizes phant_gpu_snap_size reports
    uint32_t snp_n = 0, snp_m = 0;
    uint64_t snp_ea = 0, snp_ab = 0, snp_ns = 0, snp_es = 0, snp_sb = 0, snp_refs = 0;
    // contract code (DESIGN.md §4.3i): rows sorted by codeHash, ping-pong across merges, and the arena they point into; only
    // put_codes, prune_codes and close change them
    DevBuf code_rows[2], code_arena;
    int cc = 0;
    uint32_t n_codes = 0;
    uint64_t code_used = 0, code_bytes = 0; // arena bytes in use (16-byte aligned entries); the held codes' lengths
    // the current tables: the ping-pong buffers in use, and the account trie's value arena
    AccRow* acc_rows() const { return (AccRow*)A[ac].ptr; }
    SlotRow* slot_table() const { return (SlotRow*)S[sc].ptr; }
    const KRow* acct_rows() const { return (const KRow*)acct_sp.rows[acct_sp.cur].ptr; }
    const uint8_t* acct_arena() const { return (const uint8_t*)acct_sp.arena.ptr; }
    // the node set in wit_res (empty when wit_n is 0) with its digests (nullable), as the chain walks read it
    tn::PcSet node_set(const uint8_t* digests) const
    {
        const uint64_t* off = wit_n ? (const uint64_t*)wit_res.ptr : nullptr;
        return tn::PcSet{off ? (const uint8_t*)(off + wit_n + 1) : nullptr, off, digests, (uint32_t)wit_n};
    }
    void drop_result()
    {
        wit_res.release();
        prf_res.release();
        tnd_res.release();
        snp_res.release();
        held = Result::NONE;
        wit_n = wit_bytes = prf_refs = tnd_nodes = tnd_bytes = 0;
        snp_ea = snp_ab = snp_ns = snp_es = snp_sb = snp_refs = 0;
    }
    std::vector<DevBuf*> bufs()
    {
        std::vector<DevBuf*> v = {&S[0], &S[1], &A[0], &A[1], &pool[0], &pool[1], &in, &dirty, &work, &forest, &sort, &acct_sp.rows[0], &acct_sp.rows[1],
                &acct_sp.arena, &acct_sp.top, &acct_sp.present, &acct_sp.dirty, &acct_sp.buckets, &acct_sp.gather, &acct_sp.gvals, &acct_sp.sort,
                &wit_out, &wit_res, &prf_res, &tnd_res, &snp_res, &code_rows[0], &code_rows[1], &code_arena};
        for (DevBuf* b : journal_bufs()) v.push_back(b);
        return v;
    }
    std::vector<DevBuf*> journal_bufs()
    {
        std::vector<DevBuf*> v = {&next.buf};
        for (Record& r : journal) v.push_back(&r.buf);
        for (DevBuf& b : spare) v.push_back(&b);
        return v;
    }
};

namespace {

using RsResult = phant_gpu_resident_state::Result;

// none of `ps` is a device pointer (a null one is not): the calls that take host arrays refuse device ones
bool host_ptrs(std::initializer_list<const void*> ps)
{
    for (const void* p : ps) {
        if (!p) continue;
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); continue; }
        if (a.type == cudaMemoryTypeDevice) return false;
    }
    return true;
}

// cannot happen: the account trie's leaves are written by account_fill_kernel
int rs_undecodable_leaf(phant_gpu_ctx* ctx)
{
    snprintf(ctx->last_error, sizeof ctx->last_error, "resident state: an account leaf of the account trie does not decode");
    return PHANT_GPU_E_CUDA;
}

// a diff on the device: na accounts, ms slots; the layout of the staging area and of an undo record
struct RsDiff {
    uint8_t* akeys; uint8_t* aflags; uint64_t* nonce; uint8_t* bal; uint8_t* code;
    uint32_t* sacc; uint8_t* skeys; uint8_t* svals;
    uint32_t na, ms;
    void take(Carve& c, uint32_t n_accounts, uint32_t n_slots)
    {
        na = n_accounts;
        ms = n_slots;
        akeys = c.take<uint8_t>(32ull * na); aflags = c.take<uint8_t>(na); nonce = c.take<uint64_t>(na);
        bal = c.take<uint8_t>(32ull * na); code = c.take<uint8_t>(32ull * na);
        sacc = c.take<uint32_t>(ms); skeys = c.take<uint8_t>(32ull * ms); svals = c.take<uint8_t>(32ull * ms);
    }
};

// A checked host diff copied to the device, into the arrays of `dd` (laid out by RsDiff::take in the caller's area).
int stage_diff(phant_gpu_ctx* ctx, const phant_gpu_state_diff* d, const RsDiff& dd)
{
    cudaStream_t s = ctx->stream;
    const uint32_t na = dd.na, ms = dd.ms;
    CU(cudaMemcpyAsync(dd.akeys, d->account_keys32, 32ull * na, cudaMemcpyHostToDevice, s));
    if (d->account_flags) CU(cudaMemcpyAsync(dd.aflags, d->account_flags, na, cudaMemcpyHostToDevice, s));
    else CU(cudaMemsetAsync(dd.aflags, 0, na, s));
    CU(cudaMemcpyAsync(dd.nonce, d->nonce, 8ull * na, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dd.bal, d->balance32, 32ull * na, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dd.code, d->code_hash32, 32ull * na, cudaMemcpyHostToDevice, s));
    if (ms) {
        CU(cudaMemcpyAsync(dd.sacc, d->slot_account, 4ull * ms, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dd.skeys, d->slot_keys32, 32ull * ms, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dd.svals, d->slot_vals32, 32ull * ms, cudaMemcpyHostToDevice, s));
    }
    ctx->stats.h2d_bytes += 32ull * na * 3 + 9ull * na + 68ull * ms;
    return PHANT_GPU_OK;
}

// Host-side checks of a diff that the resident apply and the transition roots share (nothing is launched on a bad argument):
// host pointers only, sizes, flag bits, slot owners.
int check_diff_host(phant_gpu_ctx* ctx, const phant_gpu_state_diff* d)
{
    const uint64_t na64 = d->n_accounts, ms64 = d->n_slots;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // host tables only, as kind 1
    if (na64 >= (1ull << 28) || ms64 >= (1ull << 28)) return PHANT_GPU_E_INVALID;
    if (na64 && (!d->account_keys32 || !d->nonce || !d->balance32 || !d->code_hash32)) return PHANT_GPU_E_INVALID;
    if (ms64 && (!d->slot_account || !d->slot_keys32 || !d->slot_vals32)) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({d->account_keys32, d->account_flags, d->nonce, d->balance32, d->code_hash32, d->slot_account, d->slot_keys32, d->slot_vals32}))
        return PHANT_GPU_E_INVALID;
    const uint32_t na = (uint32_t)na64, ms = (uint32_t)ms64;
    if (d->account_flags)
        for (uint32_t i = 0; i < na; ++i)
            if (d->account_flags[i] & ~(PHANT_GPU_ACCOUNT_DELETE | PHANT_GPU_ACCOUNT_CLEAR_STORAGE)) return PHANT_GPU_E_INVALID;
    for (uint32_t j = 0; j < ms; ++j) {
        const uint32_t a = d->slot_account[j];
        if (a >= na || (d->account_flags && (d->account_flags[a] & PHANT_GPU_ACCOUNT_DELETE))) return PHANT_GPU_E_INVALID;
    }
    return PHANT_GPU_OK;
}

// A host diff for the apply or the witness: checked against the resident tables' bounds and by check_diff_host, then staged
// into st->in (nothing resident changes).  A diff with no account (it has no slot either) is checked but not staged: dd.na == 0.
int rs_stage(phant_gpu_resident_state* st, const phant_gpu_state_diff* d, RsDiff& dd)
{
    phant_gpu_ctx* ctx = st->ctx;
    const uint64_t na64 = d->n_accounts, ms64 = d->n_slots;
    if (st->nA + na64 >= (1ull << 30) || st->nS + ms64 >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    RC(check_diff_host(ctx, d));
    dd = RsDiff{};
    if (na64 == 0) return PHANT_GPU_OK;
    RC(carve(ctx, st->in, [&](Carve& c) { dd.take(c, (uint32_t)na64, (uint32_t)ms64); }));
    return stage_diff(ctx, d, dd);
}

// A staged diff sorted and its accounts classified against the account rows, for the apply and the witness alike; laid out by
// take() inside the caller's carve of st->dirty.  The accounts are sorted by key (perm_a, rank) into rows and flags; the slots
// by (account rank, key) into rows and flags.  del_flag / ins_at (nA + 3 each) are the account merge's.  counters[0..1]: an
// account twice, an (account, slot) pair twice; counters[6..7]: account rows inserted, deleted.
struct RsSorted {
    uint32_t *perm_a, *rank, *alb, *ains, *seg, *perm_s, *sacc, *del_flag, *ins_at, *counters;
    uint8_t *adel, *aclear, *akind, *sdel, *sabs;
    AccRow* arows;
    SlotRow* srows;
    void take(Carve& c, uint32_t na, uint32_t ms, uint32_t nA)
    {
        perm_a = c.take<uint32_t>(na); rank = c.take<uint32_t>(na); arows = c.take<AccRow>(na);
        adel = c.take<uint8_t>(na); aclear = c.take<uint8_t>(na); akind = c.take<uint8_t>(na); alb = c.take<uint32_t>(na); ains = c.take<uint32_t>(na);
        seg = c.take<uint32_t>(ms); perm_s = c.take<uint32_t>(ms); srows = c.take<SlotRow>(ms); sacc = c.take<uint32_t>(ms);
        sdel = c.take<uint8_t>(ms); sabs = c.take<uint8_t>(ms);
        del_flag = c.take<uint32_t>(nA + 3); ins_at = c.take<uint32_t>(nA + 3);
        counters = c.take<uint32_t>(16);
    }
};

// Enqueues the sort and the account classification of `dd` into `f`; reads nothing back.
int rs_sort_classify(phant_gpu_resident_state* st, const RsDiff& dd, const RsSorted& f)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t na = dd.na, ms = dd.ms, nA = st->nA;
    CU(cudaMemsetAsync(f.counters, 0, 64, s));
    CU(cudaMemsetAsync(f.del_flag, 0, 4ull * (nA + 3), s));
    CU(cudaMemsetAsync(f.ins_at, 0, 4ull * (nA + 3), s));
    RC(sort_by_segment_and_hash(ctx, dd.akeys, nullptr, na, f.perm_a, st->sort));
    rs_rank_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(f.perm_a, na, f.rank);
    rs_acc_dirty_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(dd.akeys, dd.aflags, f.perm_a, na, f.arows, f.adel, f.aclear, f.counters);
    ctx->stats.launches += 2;
    if (ms) {
        gather_u32_kernel<<<grid1d(dev, ms, 256), 256, 0, s>>>(f.rank, dd.sacc, ms, f.seg);
        RC(sort_by_segment_and_hash(ctx, dd.skeys, f.seg, ms, f.perm_s, st->sort));
        rs_slot_dirty_kernel<<<grid1d(dev, ms, 256), 256, 0, s>>>(dd.akeys, dd.aflags, dd.sacc, dd.skeys, dd.svals, f.seg, f.perm_s, ms, f.srows,
                                                                  f.sacc, f.sdel, f.sabs, f.counters);
        ctx->stats.launches += 2;
    }
    rs_classify_kernel<AccRow, 32><<<grid1d(dev, na, 128), 128, 0, s>>>(st->acc_rows(), nA, f.arows, na, f.adel, nullptr, f.alb,
                                                                       f.akind, f.del_flag, f.ins_at, f.ains, f.counters + 6);
    ctx->stats.launches++;
    return PHANT_GPU_OK;
}

// An apply from a diff already on the device: sort, check, classify, capture the undo record (rec non-null), merge, rebuild.
int rs_core(phant_gpu_resident_state* st, const RsDiff& dd, phant_gpu_resident_state::Record* rec, uint8_t out_root[32], uint8_t* storage_roots32)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t na = dd.na, ms = dd.ms, nS = st->nS, nA = st->nA;
    const uint8_t* akeys = dd.akeys;
    const uint8_t* aflags = dd.aflags;
    const uint64_t* nonce = dd.nonce;
    const uint8_t* bal = dd.bal;
    const uint8_t* code = dd.code;

    const uint32_t nmax = (nS > nA ? nS : nA) + 3;
    RsSorted f;
    uint32_t *ains_index, *slb, *sins, *sins_index, *mw, *ains_cnt;
    uint32_t *u_listed, *u_apos, *u_nslots, *u_soff, *up_flag, *up_pos, *idx;
    uint8_t *skind, *sroot_out;
    Plan p;
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        f.take(c, na, ms, nA);
        ains_index = c.take<uint32_t>(na + 2);
        skind = c.take<uint8_t>(ms);
        slb = c.take<uint32_t>(ms);
        sins = c.take<uint32_t>(ms + 2);
        sins_index = c.take<uint32_t>(ms + 2);
        mw = c.take<uint32_t>(nmax * 5ull); // merge work: del_flag, ins_at, keep, K, I
        p.row = c.take<uint32_t>(na + 2); p.dlo = c.take<uint32_t>(na + 2); p.dhi = c.take<uint32_t>(na + 2); p.viol = c.take<uint32_t>(na + 2);
        p.L = c.take<uint8_t>(na); p.full = c.take<uint8_t>(na); p.active = c.take<uint8_t>(na);
        sroot_out = c.take<uint8_t>(32ull * na);
        ains_cnt = c.take<uint32_t>(na);
        u_listed = c.take<uint32_t>(rec ? na + 2 : 0); // undo record: listed accounts, their positions, slots, slot offsets
        u_apos = c.take<uint32_t>(rec ? na + 2 : 0);
        u_nslots = c.take<uint32_t>(rec ? na + 2 : 0);
        u_soff = c.take<uint32_t>(rec ? na + 2 : 0);
        up_flag = c.take<uint32_t>(na + 2); // upserted flags, their positions, the index: upserted then deleted, each in the diff's order
        up_pos = c.take<uint32_t>(na + 2);
        idx = c.take<uint32_t>(na);
    }));
    uint32_t* del_flag = mw; // the slot merge's; del_flag and ins_at first: one memset clears both
    uint32_t* ins_at = mw + nmax;
    uint32_t* keep = mw + 2ull * nmax;
    uint32_t* Ksc = mw + 3ull * nmax;
    uint32_t* Isc = mw + 4ull * nmax;
    uint32_t* counters = f.counters; // classification: accounts [6..7], slots [8..9], dropped slots [2], pool layout [3]
    unsigned long long* pool_bound = (unsigned long long*)(counters + 10); // counters[10..11]
    RC(rs_sort_classify(st, dd, f));
    rs_up_flag_kernel<<<grid1d(dev, na + 1, 256), 256, 0, s>>>(aflags, na, up_flag);
    RC(scan_u32(ctx, up_flag, up_pos, na + 1));
    rs_partition_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(up_flag, up_pos, na, idx);
    ctx->stats.launches += 2;
    uint32_t hc[16];
    CU(cudaMemcpyAsync(hc, counters, 64, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(hc + 15, up_pos + na, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (hc[0] || hc[1]) return PHANT_GPU_E_INVALID; // an account twice, or (account, slot) twice
    const uint32_t n_up = hc[15], n_del = na - n_up;
    const uint32_t a_ins = hc[6], a_del = hc[7], nA_new = nA + a_ins - a_del;
    CU(cudaMemsetAsync(mw, 0, 4ull * nmax * 2, s));
    if (ms) {
        rs_classify_kernel<SlotRow, 64><<<grid1d(dev, ms, 128), 128, 0, s>>>(st->slot_table(), nS, f.srows, ms, f.sdel, f.sabs, slb,
                                                                            skind, del_flag, ins_at, sins, counters + 8);
        ctx->stats.launches++;
    }
    rs_clear_slots_kernel<<<grid1d(dev, na, 256, 32), 256, 0, s>>>(st->slot_table(), nS, st->acc_rows(), f.arows,
                                                                   f.aclear, f.akind, f.alb, na, del_flag, counters);
    CU(cudaMemsetAsync(ains_cnt, 0, 4ull * na, s));
    if (ms) rs_slot_ins_count_kernel<<<grid1d(dev, ms, 256), 256, 0, s>>>(f.sacc, skind, ms, ains_cnt);
    rs_pool_bound_kernel<<<grid1d(dev, na, 128), 128, 0, s>>>(st->slot_table(), nS, st->acc_rows(), f.arows,
                                                             f.adel, f.aclear, f.akind, f.alb, ains_cnt, na, pool_bound);
    ctx->stats.launches += ms ? 3 : 2;
    const KRow* krows = st->acct_rows();
    const uint8_t* karena = st->acct_arena();
    if (rec) { // the undo record's size; counters[12]: an old account body that does not decode
        rs_undo_size_kernel<<<grid1d(dev, na + 1, 128), 128, 0, s>>>(f.arows, f.aclear, f.akind, f.alb, na, st->slot_table(), nS,
                                                                     f.sacc, ms, krows, karena, u_listed, u_nslots, counters + 12);
        RC(scan_u32(ctx, u_listed, u_apos, na + 1));
        RC(scan_u32(ctx, u_nslots, u_soff, na + 1));
        ctx->stats.launches++;
    }
    CU(cudaMemcpyAsync(hc, counters, 64, cudaMemcpyDeviceToHost, s));
    if (rec) {
        CU(cudaMemcpyAsync(hc + 13, u_apos + na, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(hc + 14, u_soff + na, 4, cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    if (rec && hc[12]) return rs_undecodable_leaf(ctx);
    const uint32_t s_ins = hc[8], s_del = hc[9] + hc[2], nS_new = nS + s_ins - s_del;
    const uint64_t pool_max = st->pool_nodes + ((uint64_t)hc[11] << 32 | hc[10]);
    // ---- the resident tables, the pool this apply may re-lay out into, and the account trie's next row table and update area
    // (staging + classify / merge scratch) are reserved before the first write; scratch sized by what the merge leaves (the forest inputs) is reserved later,
    // and a failure from there on marks the state failed (phant_gpu_resident_state_apply) ----
    const bool s_merge = s_ins || s_del, a_merge = a_ins || a_del;
    if (s_merge) RC(st->S[1 - st->sc].reserve(ctx, 96ull * nS_new + 256));
    if (a_merge) RC(st->A[1 - st->ac].reserve(ctx, 80ull * nA_new + 256));
    RC(st->pool[1 - st->pc].reserve(ctx, 33ull * pool_max + 64));
    RC(st->acct_sp.rows[1 - st->acct_sp.cur].reserve(ctx, sizeof(KRow) * (st->acct_sp.n + na) + 64));
    {
        StrieDirty area; // account leaves are at most 110 bytes
        RC(strie_dirty_area(ctx, st->acct_sp, na, 112ull * na, &area));
    }
    if (rec) { // the undo record: a diff in the staging layout, then the old storage roots, filled from the tables as they are before the merge
        RsDiff r;
        uint8_t* rsroot;
        RC(carve(ctx, rec->buf, [&](Carve& c) { r.take(c, hc[13], hc[14]); rsroot = c.take<uint8_t>(32ull * hc[13]); }));
        rs_undo_fill_kernel<<<grid1d(dev, na, 256, 32), 256, 0, s>>>(f.arows, f.aclear, f.akind, f.alb, na, st->slot_table(), nS,
                                                                   f.srows, f.sacc, skind, slb, ms, krows, karena, u_apos, u_soff, r.akeys,
                                                                   r.aflags, r.nonce, r.bal, r.code, r.sacc, r.skeys, r.svals);
        rs_undo_sroot_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(f.arows, f.akind, f.alb, na, krows, karena, u_apos, rsroot);
        ctx->stats.launches += 2;
        rec->na = r.na;
        rec->ms = r.ms;
    }
    st->writing = true; // from here on a failure leaves the tables half-updated

    // ---- merge both tables ----
    if (ms) {
        rs_replace_kernel<SlotRow><<<grid1d(dev, ms, 256), 256, 0, s>>>(f.srows, skind, slb, ms, st->slot_table());
        ctx->stats.launches++;
    }
    if (s_merge) RC(rs_merge<SlotRow>(ctx, st->S, st->sc, nS, f.srows, ms, skind, slb, sins, del_flag, ins_at, keep, Ksc, Isc, sins_index));
    if (a_merge) RC(rs_merge<AccRow>(ctx, st->A, st->ac, nA, f.arows, na, f.akind, f.alb, f.ains, f.del_flag, f.ins_at, keep, Ksc, Isc, ains_index));
    st->nS = nS_new;
    st->nA = nA_new;
    AccRow* A = st->acc_rows();
    const SlotRow* S = st->slot_table();

    // ---- storage roots: rounds of (plan, pool layout, dirty buckets as one forest, dense levels); a round after the first
    // only rebuilds the accounts whose dense top broke the premise, one level lower ----
    bool layout = hc[3] != 0;
    for (uint32_t round = 0;; ++round) {
        CU(cudaMemsetAsync(counters, 0, 64, s));
        if (!round) CU(cudaMemsetAsync(p.viol, 0, 4ull * na, s));
        rs_plan_kernel<<<grid1d(dev, na, 128), 128, 0, s>>>(A, st->nA, S, st->nS, f.arows, f.adel, f.aclear, f.akind, f.sacc, ms, na, round, p,
                                                            counters);
        CU(cudaMemsetAsync(p.viol, 0, 4ull * na, s)); // the plan has read the last round's flags
        uint32_t *first, *F, *cnt, *off;
        RC(carve(ctx, st->work, [&](Carve& c) {
            first = c.take<uint32_t>(ms + 2); F = c.take<uint32_t>(ms + 2); cnt = c.take<uint32_t>(na + 2); off = c.take<uint32_t>(na + 2);
        }));
        rs_slot_first_kernel<<<grid1d(dev, ms + 1, 256), 256, 0, s>>>(f.srows, f.sacc, ms, p, first);
        RC(scan_u32(ctx, first, F, ms + 1));
        rs_bucket_count_kernel<<<grid1d(dev, na + 1, 256), 256, 0, s>>>(F, na, p, cnt);
        RC(scan_u32(ctx, cnt, off, na + 1));
        CU(cudaMemcpyAsync(hc, counters, 64, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(hc + 15, off + na, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches += 3;
        const uint32_t E = hc[15], maxL = hc[5];
        layout = layout || hc[3];
        if (layout) { // new region offsets for every account row; regions still valid are copied over
            uint64_t *size, *nbase;
            RC(carve(ctx, st->forest, [&](Carve& c) { size = c.take<uint64_t>(st->nA + 2); nbase = c.take<uint64_t>(st->nA + 2); }));
            rs_pool_size_kernel<<<grid1d(dev, st->nA, 256), 256, 0, s>>>(A, st->nA, size);
            RC(scan_sizes(ctx, size, nbase, st->nA));
            uint64_t nodes = 0;
            CU(cudaMemcpyAsync(&nodes, nbase + st->nA, 8, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            const int nxt = 1 - st->pc;
            if (33ull * nodes + 64 > st->pool[nxt].cap) return PHANT_GPU_E_CUDA; // cannot happen: pool_max bounds it
            uint8_t* otop = (uint8_t*)st->pool[st->pc].ptr;
            rs_pool_move_kernel<<<grid1d(dev, st->nA, 256, 32), 256, 0, s>>>(A, st->nA, nbase, otop, otop + 32 * st->pool_nodes,
                                                                           (uint8_t*)st->pool[nxt].ptr, (uint8_t*)st->pool[nxt].ptr + 32 * nodes);
            ctx->stats.launches += 2;
            st->pc = nxt;
            st->pool_nodes = nodes;
            layout = false;
        }
        uint8_t* top = (uint8_t*)st->pool[st->pc].ptr;
        uint8_t* present = top + 32 * st->pool_nodes;
        if (E) {
            uint32_t *e_acc, *e_b, *lo, *ecnt, *seg_off, *estart, *nfirst, *npos, *npar, *nbase, *nown;
            uint8_t* roots;
            RC(carve(ctx, st->forest, [&](Carve& c) {
                e_acc = c.take<uint32_t>(E); e_b = c.take<uint32_t>(E);
                lo = c.take<uint32_t>(E + 2); ecnt = c.take<uint32_t>(E + 2); seg_off = c.take<uint32_t>(E + 2); estart = c.take<uint32_t>(E + 2);
                roots = c.take<uint8_t>(32ull * E);
                nfirst = c.take<uint32_t>(E + 2); npos = c.take<uint32_t>(E + 2); // node lists of one level
                npar = c.take<uint32_t>(E + 2); nbase = c.take<uint32_t>(E + 2); nown = c.take<uint32_t>(E + 2);
            }));
            rs_fill_entries_kernel<<<grid1d(dev, ms > na ? ms : na, 256, 32), 256, 0, s>>>(f.srows, f.sacc, ms, first, F, off, na, p, e_acc, e_b);
            rs_entry_range_kernel<<<grid1d(dev, E + 1, 128), 128, 0, s>>>(S, st->nS, A, e_acc, e_b, E, p, lo, ecnt, estart);
            RC(scan_u32(ctx, ecnt, seg_off, E + 1));
            uint32_t mk = 0;
            CU(cudaMemcpyAsync(&mk, seg_off + E, 4, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            ctx->stats.launches += 2;
            if (mk) {
                uint32_t *unit, *seg_of_key, *fko;
                uint8_t *fk, *fv;
                uint64_t *fvs, *fvo;
                RC(carve(ctx, st->sort, [&](Carve& g) {
                    unit = g.take<uint32_t>(mk); seg_of_key = g.take<uint32_t>(mk + 1); fk = g.take<uint8_t>(32ull * mk); fko = g.take<uint32_t>(mk + 1);
                    fvs = g.take<uint64_t>(mk + 2); fvo = g.take<uint64_t>(mk + 2); fv = g.take<uint8_t>(33ull * mk);
                }));
                const uint8_t* srow = (const uint8_t*)S;
                rs_gather_kernel<<<grid1d(dev, E, 256, 32), 256, 0, s>>>(lo, seg_off, E, unit, seg_of_key);
                storage_value_size_kernel<<<grid1d(dev, mk, 256), 256, 0, s>>>(srow + 64, unit, mk, fvs);
                RC(scan_sizes(ctx, fvs, fvo, mk));
                storage_fill_kernel<<<grid1d(dev, mk + 1, 256), 256, 0, s>>>(srow + 32, srow + 64, unit, mk, fvo, fk, fko, fv);
                ctx->stats.launches += 3;
                RC(build_forest(ctx, {.keys = fk, .key_off = fko, .vals = fv, .val_off = fvo, .n = mk, .seg_off = seg_off, .n_seg = E,
                                      .seg_of_key = seg_of_key, .roots = roots, .slot_stride = /*32-byte keys, values <= 33 B*/ 96, .seg_start = estart}));
            } else {
                RC(build_forest(ctx, {.seg_off = seg_off, .n_seg = E, .roots = roots})); // every listed bucket empty
            }
            rs_scatter_roots_kernel<<<grid1d(dev, E, 256), 256, 0, s>>>(roots, e_acc, e_b, ecnt, E, p, A, top, present);
            ctx->stats.launches++;
            RC(fr_opt_in(ctx));
            for (int dd = (int)maxL - 1; dd >= 0; --dd) { // one launch per level across all accounts
                rs_node_flag_kernel<<<grid1d(dev, E + 1, 256), 256, 0, s>>>(e_acc, e_b, E, (uint32_t)dd, p, nfirst);
                RC(scan_u32(ctx, nfirst, npos, E + 1));
                rs_node_list_kernel<<<grid1d(dev, E, 256), 256, 0, s>>>(e_acc, e_b, nfirst, npos, E, (uint32_t)dd, p, A, npar, nbase, nown);
                st_top_branch_kernel<<<fr_grid(dev, E), FR_WARPS * 32, FR_SMEM, s>>>(
                    top + 32 * level_base(dd + 1), present + level_base(dd + 1), npar, nbase, nown, E, npos + E, top + 32 * level_base(dd),
                    present + level_base(dd), p.viol);
                ctx->stats.launches += 4;
            }
            rs_top_root_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(na, p, A, top, present);
            ctx->stats.launches++;
        }
        // premise check of this round: any listed account whose dense top has a one-child node
        RC(cub_call(ctx, [&](void* tmp, size_t& b) { return cub::DeviceReduce::Max(tmp, b, p.viol, counters + 4, (int64_t)na, s); }));
        uint32_t any = 0;
        CU(cudaMemcpyAsync(&any, counters + 4, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches++;
        if (!any) break;
        if (round > 8) return PHANT_GPU_E_CUDA; // cannot happen: every round lowers L of the accounts it rebuilds
    }
    rs_roots_out_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(f.perm_a, na, p, A, sroot_out);
    ctx->stats.launches++;

    // ---- account leaves, encoded by S's account encoder from the new storage roots, into the account trie ----
    uint32_t* ako;
    uint64_t *avs, *avo;
    RC(carve(ctx, st->work, [&](Carve& c) { avs = c.take<uint64_t>(n_up + 2); avo = c.take<uint64_t>(n_up + 2); ako = c.take<uint32_t>(n_up + 2); }));
    uint64_t vb = 0;
    if (n_up) {
        account_size_kernel<<<grid1d(dev, n_up, 256), 256, 0, s>>>(nonce, bal, idx, n_up, avs);
        RC(scan_sizes(ctx, avs, avo, n_up));
        CU(cudaMemcpyAsync(&vb, avo + n_up, 8, cudaMemcpyDeviceToHost, s));
        ctx->stats.launches++;
    }
    CU(cudaStreamSynchronize(s)); // vb, read back above, sizes the update area
    StrieDirty area;
    RC(strie_dirty_area(ctx, st->acct_sp, na, vb, &area));
    if (n_up) {
        account_fill_kernel<<<grid1d(dev, n_up + 1, 256), 256, 0, s>>>(nonce, bal, sroot_out, code, akeys, idx, n_up, avo, area.keys, ako, area.vals);
        ctx->stats.launches++;
    } else CU(cudaMemsetAsync(avo, 0, 8, s));
    if (n_del) {
        gather_rows32_kernel<<<grid1d(dev, n_del, 256), 256, 0, s>>>(akeys, idx + n_up, n_del, area.keys + 32ull * n_up);
        ctx->stats.launches++;
    }
    rs_acc_voff_kernel<<<grid1d(dev, na + 1, 256), 256, 0, s>>>(avo, n_up, na, area.val_off);
    ctx->stats.launches++;
    RC(strie_apply(ctx, st->acct_sp, na, vb, out_root));
    if (storage_roots32) {
        CU(cudaMemcpyAsync(storage_roots32, sroot_out, 32ull * na, cudaMemcpyDeviceToHost, s));
        ctx->stats.d2h_bytes += 32ull * na;
        CU(cudaStreamSynchronize(s));
    }
    return PHANT_GPU_OK;
}

// The front end of witness, prove and trie_nodes: the staged keys sorted and classified (f) and the tries of their accounts
// (w), laid out first in the caller's carve of st->dirty.  rs_query_tries enqueues both; once the caller's candidate kernels
// are enqueued, rs_query_check reads the counters back into hc.
struct RsQuery {
    RsSorted f;
    WitTries w;
    uint32_t hc[16];
    void take(Carve& c, uint32_t na, uint32_t ms, uint32_t nA)
    {
        f.take(c, na, ms, nA);
        w.ok = c.take<uint8_t>(na + 1); w.L = c.take<uint32_t>(na + 1); w.base = c.take<uint32_t>(na + 1);
        w.slo = c.take<uint32_t>(na + 1); w.shi = c.take<uint32_t>(na + 1);
    }
};

int rs_query_tries(phant_gpu_resident_state* st, const RsDiff& dd, const RsQuery& rq)
{
    phant_gpu_ctx* ctx = st->ctx;
    const SparseTrie& sp = st->acct_sp;
    const RsSorted& f = rq.f;
    RC(rs_sort_classify(st, dd, f));
    wit_tries_kernel<<<grid1d(ctx->device, dd.na + 1, 128), 128, 0, ctx->stream>>>(st->acc_rows(), st->slot_table(), st->nS, f.arows, f.aclear,
                                                                                   f.akind, f.alb, dd.na, (uint32_t)sp.n, sp.L, rq.w);
    ctx->stats.launches++;
    return PHANT_GPU_OK;
}

// The counters to rq.hc (64 bytes) and, when the caller counts its proof keys on the device (d_np), that count to *np (4 bytes),
// once the caller's candidates are enqueued.  An account or an (account, slot) pair listed twice is refused.
int rs_query_check(phant_gpu_resident_state* st, RsQuery& rq, const uint32_t* d_np, uint32_t* np)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    CU(cudaMemcpyAsync(rq.hc, rq.f.counters, 64, cudaMemcpyDeviceToHost, s));
    if (d_np) CU(cudaMemcpyAsync(np, d_np, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.d2h_bytes += d_np ? 68 : 64;
    return rq.hc[0] || rq.hc[1] ? PHANT_GPU_E_INVALID : PHANT_GPU_OK;
}

// The keys step of rs_nodes for the witness and the trie nodes: the np proof keys among n candidates (ckeys, each in trie
// cseg, NONE when it is no proof key), sorted by (trie, key) into pkeys / ptrie; cperm (n) is scratch.
int rs_candidate_keys(phant_gpu_resident_state* st, const uint8_t* ckeys, const uint32_t* cseg, uint32_t* cperm, uint32_t n, uint32_t np,
                      uint8_t* pkeys, uint32_t* ptrie)
{
    phant_gpu_ctx* ctx = st->ctx;
    RC(sort_by_segment_and_hash(ctx, ckeys, cseg, n, cperm, st->sort)); // the NONE candidates sort last
    wit_proof_keys_kernel<<<grid1d(ctx->device, np, 256), 256, 0, ctx->stream>>>(ckeys, cseg, cperm, np, pkeys, ptrie);
    ctx->stats.launches++;
    return PHANT_GPU_OK;
}

// The node set of np proof keys, held in st->wit_res as CSR (st->wit_n nodes, st->wit_bytes bytes; none when np is 0): the
// back end the witness, the proofs and the trie nodes share.  keys(pkeys, ptrie) writes the keys, sorted by (trie, key) in
// the tries rq classified, into pkeys / ptrie (np each), which lie in st->work with first / bpos (np + 1 each); the dense-top
// nodes on the keys' paths are encoded from the pool, the buckets that hold a proof key are rebuilt as one forest whose nodes
// on the proof paths are exported, and the exported nodes are sorted by digest with the duplicates dropped.  digests
// (nullable) receives the kept nodes' digests, 32 bytes each in the CSR's order, in st->work (valid until its next carve).
// Only scratch is written.
template <class Keys> int rs_nodes(phant_gpu_resident_state* st, const RsQuery& rq, uint32_t np, Keys&& keys, uint8_t** digests)
{
    if (np == 0) return PHANT_GPU_OK;
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t nS = st->nS;
    const SlotRow* S = st->slot_table();
    const SparseTrie& sp = st->acct_sp;
    const KRow* krows = st->acct_rows();
    const uint32_t n = (uint32_t)sp.n;
    const RsSorted& f = rq.f;
    const WitTries& w = rq.w;
    uint8_t* pkeys;
    uint32_t *ptrie, *first, *bpos;
    RC(carve(ctx, st->work, [&](Carve& c) {
        pkeys = c.take<uint8_t>(32ull * np); ptrie = c.take<uint32_t>(np); first = c.take<uint32_t>(np + 1); bpos = c.take<uint32_t>(np + 1);
    }));
    RC(keys(pkeys, ptrie));

    // ---- the buckets that hold a proof key ----
    const uint8_t* pool_top = (const uint8_t*)st->pool[st->pc].ptr;
    const WitTops tp{(const uint8_t*)sp.top.ptr, (const uint8_t*)sp.present.ptr, pool_top, pool_top + 32 * st->pool_nodes};
    wit_bucket_flag_kernel<<<grid1d(dev, np + 1, 256), 256, 0, s>>>(pkeys, ptrie, np, w, tp, first);
    RC(scan_u32(ctx, first, bpos, np + 1));
    uint32_t E = 0;
    CU(cudaMemcpyAsync(&E, bpos + np, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches++;
    ctx->stats.d2h_bytes += 4;
    uint32_t *etrie, *elo, *ecnt, *estart, *seg_off;
    uint8_t* roots;
    RC(carve(ctx, st->forest, [&](Carve& c) {
        etrie = c.take<uint32_t>(E + 1); elo = c.take<uint32_t>(E + 1); ecnt = c.take<uint32_t>(E + 2); estart = c.take<uint32_t>(E + 1);
        seg_off = c.take<uint32_t>(E + 2); roots = c.take<uint8_t>(32ull * E + 32);
    }));
    wit_bucket_kernel<<<grid1d(dev, np + 1, 128), 128, 0, s>>>(pkeys, ptrie, np, first, bpos, w, krows, n, S, nS, f.arows, etrie, elo, ecnt, estart);
    RC(scan_u32(ctx, ecnt, seg_off, E + 1));
    uint32_t mk = 0;
    CU(cudaMemcpyAsync(&mk, seg_off + E, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches++;
    ctx->stats.d2h_bytes += 4;
    // ---- forest input: keys and leaf values of those buckets ----
    uint8_t *fk = nullptr, *fv = nullptr;
    uint32_t *fko = nullptr, *seg_of_key = nullptr, *src = nullptr;
    uint64_t *vsize = nullptr, *voff = nullptr;
    if (mk) {
        RC(carve(ctx, st->sort, [&](Carve& c) {
            fk = c.take<uint8_t>(32ull * mk); fko = c.take<uint32_t>(mk + 1); seg_of_key = c.take<uint32_t>(mk + 1); src = c.take<uint32_t>(mk);
            vsize = c.take<uint64_t>(mk + 2); voff = c.take<uint64_t>(mk + 2); fv = c.take<uint8_t>(112ull * mk); // a value is at most 110 bytes
        }));
        wit_forest_keys_kernel<<<grid1d(dev, E, 256, 32), 256, 0, s>>>(etrie, elo, seg_off, E, mk, krows, S, fk, fko, seg_of_key, src, vsize);
        RC(scan_sizes(ctx, vsize, voff, mk));
        wit_forest_vals_kernel<<<grid1d(dev, mk, 256), 256, 0, s>>>(etrie, seg_of_key, src, voff, mk, krows, st->acct_arena(), S, fv);
        ctx->stats.launches += 2;
    }

    // ---- export: dense-top nodes, then the forest's nodes on the proof paths; run again with room for all of them when the
    // output was too small (nothing differs between the runs but the capacity) ----
    uint64_t n_out = 0, need_n = 8ull * np + 64, need_b = 1536ull * np + 65536;
    ForestExport xp{pkeys, ptrie, np, etrie, seg_of_key, {}};
    for (int attempt = 0;; ++attempt) {
        WitnessOut& o = xp.out;
        RC(carve(ctx, st->wit_out, [&](Carve& c) {
            o.used = (unsigned long long*)c.take<uint64_t>(2); o.nodes = c.take<WNode>(need_n); o.digests = c.take<uint8_t>(32ull * need_n);
            o.bytes = c.take<uint8_t>(need_b);
        }));
        o.cap_nodes = need_n;
        o.cap_bytes = need_b;
        CU(cudaMemsetAsync(o.used, 0, 16, s));
        wit_dense_kernel<<<grid1d(dev, np, 128), 128, 0, s>>>(pkeys, ptrie, np, w, tp, o);
        ctx->stats.launches++;
        if (mk) RC(build_forest(ctx, {.keys = fk, .key_off = fko, .vals = fv, .val_off = voff, .n = mk, .seg_off = seg_off, .n_seg = E,
                                      .seg_of_key = seg_of_key, .roots = roots, .seg_start = estart, .xp = &xp}));
        uint64_t used[2];
        CU(cudaMemcpyAsync(used, o.used, 16, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.d2h_bytes += 16;
        n_out = used[0];
        if (used[0] <= need_n && used[1] <= need_b) break;
        if (attempt) return PHANT_GPU_E_CUDA; // cannot happen: the second run has room for what the first one counted
        need_n = used[0] > need_n ? used[0] : need_n;
        need_b = used[1] > need_b ? used[1] : need_b;
    }

    // ---- sort by digest, drop duplicates, write the CSR ----
    const uint32_t ne = (uint32_t)n_out;
    uint32_t *perm, *keep, *kidx;
    uint64_t *size, *offs;
    uint8_t* udig;
    RC(carve(ctx, st->work, [&](Carve& c) {
        perm = c.take<uint32_t>(ne + 1); keep = c.take<uint32_t>(ne + 2); kidx = c.take<uint32_t>(ne + 2);
        size = c.take<uint64_t>(ne + 2); offs = c.take<uint64_t>(ne + 2);
        udig = c.take<uint8_t>(digests ? 32ull * ne : 0);
    }));
    RC(sort_by_segment_and_hash(ctx, xp.out.digests, nullptr, ne, perm, st->sort));
    wit_unique_kernel<<<grid1d(dev, ne + 1, 256), 256, 0, s>>>(xp.out.digests, xp.out.nodes, perm, ne, keep, size);
    RC(scan_u32(ctx, keep, kidx, ne + 1));
    RC(scan_sizes(ctx, size, offs, ne));
    uint32_t nn = 0;
    uint64_t nb = 0;
    CU(cudaMemcpyAsync(&nn, kidx + ne, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&nb, offs + ne, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.d2h_bytes += 12;
    RC(st->wit_res.reserve(ctx, 8ull * (nn + 1) + nb + 256));
    uint64_t* node_off = (uint64_t*)st->wit_res.ptr;
    wit_write_kernel<<<grid1d(dev, ne, 256, 32), 256, 0, s>>>(xp.out.bytes, xp.out.nodes, perm, keep, kidx, offs, ne, node_off,
                                                              (uint8_t*)(node_off + nn + 1));
    ctx->stats.launches += 2;
    if (digests) {
        prf_digest_kernel<<<grid1d(dev, ne, 256), 256, 0, s>>>(xp.out.digests, perm, keep, kidx, ne, udig);
        ctx->stats.launches++;
        *digests = udig;
    }
    CU(cudaStreamSynchronize(s));
    st->wit_n = nn;
    st->wit_bytes = nb;
    return PHANT_GPU_OK;
}

// The pre-state witness of a diff (phant_gpu_resident_state_witness), the node set in st->wit_res.  The diff is staged and
// goes through the query front end; the proof keys of every trie (listed keys, and the surviving neighbours of deleted ones,
// counted in counters[2]; none in the empty state) are listed as candidates and handed to rs_nodes.  Only scratch is written.
int rs_witness(phant_gpu_resident_state* st, const phant_gpu_state_diff* d)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    RsDiff dd;
    RC(rs_stage(st, d, dd));
    if (dd.na == 0) return PHANT_GPU_OK;
    const uint32_t na = dd.na, ms = dd.ms;
    const uint32_t C = 3 * na + 3 * ms; // proof-key candidates
    RsQuery rq;
    uint32_t *cseg, *cperm;
    uint8_t* ckeys;
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        rq.take(c, na, ms, st->nA);
        ckeys = c.take<uint8_t>(32ull * C); cseg = c.take<uint32_t>(C); cperm = c.take<uint32_t>(C);
    }));
    RC(rs_query_tries(st, dd, rq));
    const RsSorted& f = rq.f;
    wit_acc_keys_kernel<<<grid1d(dev, na, 128), 128, 0, s>>>(f.arows, f.adel, na, st->acct_rows(), (uint32_t)st->acct_sp.n, ckeys, cseg,
                                                             f.counters + 2);
    ctx->stats.launches++;
    if (ms) {
        wit_slot_keys_kernel<<<grid1d(dev, ms, 128), 128, 0, s>>>(f.srows, f.sacc, f.sdel, ms, st->slot_table(), st->nS, rq.w, 3 * na, ckeys,
                                                                  cseg, f.counters + 2);
        ctx->stats.launches++;
    }
    RC(rs_query_check(st, rq, nullptr, nullptr));
    const uint32_t np = rq.hc[2];
    return rs_nodes(st, rq, np, [&](uint8_t* pkeys, uint32_t* ptrie) { return rs_candidate_keys(st, ckeys, cseg, cperm, C, np, pkeys, ptrie); },
                    nullptr);
}

} // namespace

namespace {
int rs_refuse_failed(phant_gpu_resident_state* st)
{
    snprintf(st->ctx->last_error, sizeof st->ctx->last_error, "resident state unusable: an earlier apply failed after it began to write");
    return PHANT_GPU_E_CUDA;
}

// The entry rule of the calls that work on the device: a null state is invalid, a state whose apply failed after it began to
// write refuses every call, and otherwise the context's device is made current.
int rs_enter(phant_gpu_resident_state* st)
{
    if (!st) return PHANT_GPU_E_INVALID;
    if (st->failed) return rs_refuse_failed(st);
    phant_gpu_ctx* ctx = st->ctx;
    CU(cudaSetDevice(ctx->device));
    return PHANT_GPU_OK;
}

// The entry rule of the calls that build a result to hold (witness, prove, trie_nodes, snap_ranges): rs_enter, the result held
// before is dropped and *out zeroed, then body() builds the new one, which is held as `kind` when it succeeds and dropped when
// it fails.
template <class Out, class Body> int rs_build_result(phant_gpu_resident_state* st, RsResult kind, Out* out, Body&& body)
{
    RC(rs_enter(st));
    st->drop_result();
    memset(out, 0, sizeof *out);
    const int rc = body();
    if (rc) {
        st->drop_result();
        return rc;
    }
    st->held = kind;
    return PHANT_GPU_OK;
}

// The copy rule of the held results, once the caller has checked that its kind is held and its arguments: every pointer in
// `host` is a host pointer (a null one is not checked), as in the requests; copy() enqueues the copies on the context's
// stream, and the call returns when they are done, with the result dropped.
template <class Copy> int rs_copy_result(phant_gpu_resident_state* st, std::initializer_list<const void*> host, Copy&& copy)
{
    if (!host_ptrs(host)) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    CU(cudaSetDevice(ctx->device));
    RC(copy());
    CU(cudaStreamSynchronize(ctx->stream));
    st->drop_result();
    return PHANT_GPU_OK;
}

// the held node set (CSR in st->wit_res) to the host: node_off[0] = 0, then the offsets and the bytes
int copy_node_set(phant_gpu_resident_state* st, uint64_t* node_off, uint8_t* nodes)
{
    node_off[0] = 0;
    if (!st->wit_n) return PHANT_GPU_OK;
    const tn::PcSet set = st->node_set(nullptr);
    RC(copy_out(st->ctx, node_off, set.off, 8ull * (st->wit_n + 1)));
    return copy_out(st->ctx, nodes, set.bytes, st->wit_bytes);
}

// Undo record r replayed onto st by the apply core, from where r lies on the device, and the root after it checked against
// the root r saved: one step of revert and of fork.  rs_core only reads the diff it is given, so r is left as it was (a fork
// replays its parent's records without consuming them).  A mismatch, or a failure after the replay's first write, leaves st
// unusable.
int rs_replay(phant_gpu_resident_state* st, const phant_gpu_resident_state::Record& r)
{
    phant_gpu_ctx* ctx = st->ctx;
    uint8_t root[32];
    memcpy(root, st->acct_sp.root, 32);
    if (r.na) {
        Carve c{(uint8_t*)r.buf.ptr};
        RsDiff d;
        d.take(c, r.na, r.ms);
        st->writing = false;
        const int rc = rs_core(st, d, nullptr, root, nullptr);
        if (rc && st->writing) st->failed = true;
        st->writing = false;
        if (rc) return rc;
    }
    if (memcmp(root, r.root, 32) != 0) { // cannot happen: the record is the exact inverse of the apply
        st->failed = true;
        snprintf(ctx->last_error, sizeof ctx->last_error, "resident state: a reverted apply did not give back the root before it");
        return PHANT_GPU_E_CUDA;
    }
    return PHANT_GPU_OK;
}
} // namespace

extern "C" int phant_gpu_resident_state_open(phant_gpu_ctx* ctx, phant_gpu_resident_state** out)
{
    if (!ctx || !out) return PHANT_GPU_E_INVALID;
    *out = nullptr;
    CU(cudaSetDevice(ctx->device));
    phant_gpu_resident_state* st = new (std::nothrow) phant_gpu_resident_state();
    if (!st) return PHANT_GPU_E_OOM;
    st->ctx = ctx;
    st->acct_sp.compact = true;
    st->acct_sp.compact_row = 112; // an account leaf is at most 110 bytes
    memcpy(st->acct_sp.root, EMPTY_ROOT_H, 32);
    *out = st;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_apply(phant_gpu_resident_state* st, const phant_gpu_state_diff* diff, uint8_t out_root[32],
                                              uint8_t* storage_roots32)
{
    if (!diff || !out_root) return PHANT_GPU_E_INVALID;
    RC(rs_enter(st));
    st->drop_result();
    st->writing = false;
    phant_gpu_resident_state::Record* rec = st->depth ? &st->next : nullptr;
    uint8_t before[32];
    memcpy(before, st->acct_sp.root, 32);
    if (rec) rec->na = rec->ms = 0;
    RsDiff dd;
    int rc = rs_stage(st, diff, dd);
    if (rc == PHANT_GPU_OK) {
        if (dd.na) rc = rs_core(st, dd, rec, out_root, storage_roots32);
        else memcpy(out_root, before, 32); // no account: nothing changes
    }
    if (rc && st->writing) st->failed = true;
    st->writing = false;
    if (rc || !rec) return rc;
    // push the record; its buffer is replaced by a spare one, and the oldest record goes once there are more than `depth`
    memcpy(rec->root, before, 32);
    st->journal.push_back(*rec);
    st->next = phant_gpu_resident_state::Record();
    if (!st->spare.empty()) { st->next.buf = st->spare.back(); st->spare.pop_back(); }
    if (st->journal.size() > st->depth) {
        st->spare.push_back(st->journal.front().buf);
        st->journal.pop_front();
    }
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_set_journal(phant_gpu_resident_state* st, uint32_t depth)
{
    if (depth > 1024) return PHANT_GPU_E_INVALID;
    RC(rs_enter(st));
    phant_gpu_ctx* ctx = st->ctx;
    CU(cudaStreamSynchronize(ctx->stream));
    st->drop_result();
    st->depth = depth;
    while (st->journal.size() > depth) {
        st->journal.front().buf.release();
        st->journal.pop_front();
    }
    for (DevBuf& b : st->spare) b.release();
    st->spare.clear();
    if (!depth) st->next.buf.release();
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_revert(phant_gpu_resident_state* st, uint32_t n_applies, uint8_t out_root[32])
{
    if (!out_root) return PHANT_GPU_E_INVALID;
    if (st && !st->failed && n_applies > st->journal.size()) return PHANT_GPU_E_INVALID; // checked before the device is set
    RC(rs_enter(st));
    st->drop_result();
    for (uint32_t k = 0; k < n_applies; ++k) { // newest first
        RC(rs_replay(st, st->journal.back()));
        st->spare.push_back(st->journal.back().buf);
        st->journal.pop_back();
    }
    memcpy(out_root, st->acct_sp.root, 32);
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// Resident world state: forks (phant_gpu_resident_state_fork, DESIGN.md §4.3l).  A fork is a new state on the same context
// holding what revert(back) would return to, built without changing the parent: the parent's live tables are copied device to
// device -- the current halves of the slot table, the account rows and the dense-top pool (references, then presence bytes,
// pool_nodes of each), and the account trie's current row table, its arena up to arena_used and its dense levels 0..L -- with
// the host scalars that describe them; then the parent's `back` newest undo records are replayed onto the copy, newest
// first, by rs_replay, read where they lie.  No scratch, held result, record or code is copied: the fork starts with journal
// depth 0 and an empty code store.
// ------------------------------------------------------------------------------------------------
namespace {
// the first n bytes of src into dst, reserved for n + pad bytes, on the context's stream (nothing when n is 0)
int copy_live(phant_gpu_ctx* ctx, DevBuf& dst, const DevBuf& src, uint64_t n, uint64_t pad)
{
    if (!n) return PHANT_GPU_OK;
    RC(dst.reserve(ctx, n + pad));
    CU(cudaMemcpyAsync(dst.ptr, src.ptr, n, cudaMemcpyDeviceToDevice, ctx->stream));
    return PHANT_GPU_OK;
}

// the live tables of st into f, a state just opened on st's context: f then holds exactly st's current state
int rs_copy_live(const phant_gpu_resident_state* st, phant_gpu_resident_state* f)
{
    phant_gpu_ctx* ctx = st->ctx;
    RC(copy_live(ctx, f->S[0], st->S[st->sc], sizeof(SlotRow) * st->nS, 256)); // the pads apply reserves with
    RC(copy_live(ctx, f->A[0], st->A[st->ac], sizeof(AccRow) * st->nA, 256));
    RC(copy_live(ctx, f->pool[0], st->pool[st->pc], 33ull * st->pool_nodes, 64));
    f->nS = st->nS;
    f->nA = st->nA;
    f->pool_nodes = st->pool_nodes;
    const SparseTrie& a = st->acct_sp;
    SparseTrie& b = f->acct_sp;
    RC(copy_live(ctx, b.rows[0], a.rows[a.cur], sizeof(KRow) * a.n, 64));
    RC(copy_live(ctx, b.arena, a.arena, a.arena_used, 64));
    if (a.n) { // an account trie with a key has its levels 0..L (st_set_L_and_rebuild_all ran when its first key came)
        const uint64_t nodes = level_base(a.L + 1);
        RC(copy_live(ctx, b.top, a.top, 32 * nodes, 64));
        RC(copy_live(ctx, b.present, a.present, nodes, 64));
    }
    b.n = a.n;
    b.arena_used = a.arena_used;
    b.L = a.L;
    memcpy(b.root, a.root, 32);
    b.updates = a.updates;
    b.rebuilds = a.rebuilds;
    b.compact = a.compact;
    b.compact_row = a.compact_row;
    CU(cudaStreamSynchronize(ctx->stream));
    return PHANT_GPU_OK;
}
} // namespace

extern "C" int phant_gpu_resident_state_fork(phant_gpu_resident_state* st, uint32_t back, phant_gpu_resident_state** out)
{
    if (!out) return PHANT_GPU_E_INVALID;
    *out = nullptr;
    if (st && !st->failed && back > st->journal.size()) return PHANT_GPU_E_INVALID; // checked before the device is set
    RC(rs_enter(st));
    phant_gpu_resident_state* f = nullptr;
    RC(phant_gpu_resident_state_open(st->ctx, &f));
    int rc = rs_copy_live(st, f);
    for (uint32_t k = 0; rc == PHANT_GPU_OK && k < back; ++k) rc = rs_replay(f, st->journal[st->journal.size() - 1 - k]); // newest first
    if (rc) {
        phant_gpu_resident_state_close(f);
        return rc;
    }
    *out = f;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_witness(phant_gpu_resident_state* st, const phant_gpu_state_diff* diff, phant_gpu_witness_size* out)
{
    if (!diff || !out) return PHANT_GPU_E_INVALID;
    RC(rs_build_result(st, RsResult::WITNESS, out, [&] { return rs_witness(st, diff); }));
    out->n_nodes = st->wit_n;
    out->nodes_bytes = st->wit_bytes;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_witness_copy(phant_gpu_resident_state* st, uint8_t* nodes, uint64_t* node_off)
{
    if (!st || st->held != RsResult::WITNESS || !node_off || (st->wit_bytes && !nodes)) return PHANT_GPU_E_INVALID;
    return rs_copy_result(st, {nodes, node_off}, [&] { return copy_node_set(st, node_off, nodes); });
}

extern "C" int phant_gpu_resident_state_root(phant_gpu_resident_state* st, uint8_t out_root[32])
{
    if (!st || !out_root) return PHANT_GPU_E_INVALID;
    if (st->failed) return rs_refuse_failed(st);
    memcpy(out_root, st->acct_sp.root, 32);
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_info(phant_gpu_resident_state* st, phant_gpu_state_info* out)
{
    if (!st || !out) return PHANT_GPU_E_INVALID;
    memset(out, 0, sizeof *out);
    out->n_accounts = st->nA;
    out->n_slots = st->nS;
    for (DevBuf* b : st->bufs()) out->device_bytes += b->cap;
    out->journal_applies = st->journal.size();
    for (DevBuf* b : st->journal_bufs()) out->journal_bytes += b->cap;
    out->n_codes = st->n_codes;
    out->code_bytes = st->code_bytes;
    return PHANT_GPU_OK;
}

extern "C" void phant_gpu_resident_state_close(phant_gpu_resident_state* st)
{
    if (!st) return;
    cudaSetDevice(st->ctx->device);
    cudaStreamSynchronize(st->ctx->stream);
    for (DevBuf* b : st->bufs()) b->release();
    delete st;
}

// ------------------------------------------------------------------------------------------------
// T: state transition roots from a witness node set and a diff (include/phant_gpu.h, DESIGN.md "T: state transition roots").
// Segments: [0, n_st) the storage tries of the listed accounts that are not deleted, then one account trie per block.  Only the
// paths of listed keys are expanded; every off-path child referenced by hash becomes a STUB (its prefix and reference), fed to
// build_forest as a leaf whose reference is cached at the depth where it hangs -- or, when the rebuild moves it up, the node it
// becomes (tr_collapsed) is encoded and hashed here and cached at its new depth.
// ------------------------------------------------------------------------------------------------
namespace {

constexpr uint32_t TB_BAD = 1, TB_MISSING = 2; // per-block flags: status 0 / status 3
enum : uint32_t { TI_LEAF = 0, TI_STUB = 1, TI_STUB_BRANCH = 2, TI_ACC = 3, TI_SLOT = 4, TI_DEL = 5 };

struct alignas(16) TFront { // a node to expand: hashed (len == 0: `ref`) or embedded (the len bytes at nodes + off)
    uint8_t prefix[32];     // the path's first `depth` nibbles, zero after
    uint8_t ref[32];
    uint64_t off;
    uint32_t len, seg, depth, lo, hi, below_ext; // [lo, hi): the sorted diff keys under it
};
struct alignas(16) TItem {
    uint8_t key[32]; // leaf / diff key; stub: its prefix, zero padded
    uint8_t ref[32]; // stub: the digest its parent holds
    uint64_t voff;   // TI_LEAF: value payload at nodes + voff; TI_ACC / TI_SLOT: index into the diff
    uint32_t vlen, seg, depth, kind;
};
struct TSeg {
    uint32_t n_st;
    const uint32_t* acc_of_seg; // n_st: the listed account of each storage segment
    const uint32_t* ablock;     // per listed account
};
__device__ __forceinline__ uint32_t seg_block(const TSeg& g, uint32_t s) { return s < g.n_st ? g.ablock[g.acc_of_seg[s]] : s - g.n_st; }
__device__ __forceinline__ void copy32(uint8_t* d, const uint8_t* s) { for (int b = 0; b < 32; ++b) d[b] = s[b]; }
__device__ __forceinline__ int cmp32(const uint8_t* a, const uint8_t* b)
{
    for (int i = 0; i < 32; ++i) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
__device__ __forceinline__ uint32_t lcp32(const uint8_t* a, const uint8_t* b)
{
    uint32_t t = 0;
    while (t < 32 && a[t] == b[t]) ++t;
    if (t == 32) return 64;
    return 2 * t + (((a[t] ^ b[t]) & 0xf0) ? 0 : 1);
}

// the diff's keys with their segments: accounts in their block's account trie, slots in their account's storage trie
__global__ void tr_diff_keys_kernel(const uint8_t* __restrict__ akeys, const uint32_t* __restrict__ ablock, uint32_t na, const uint32_t* __restrict__ sacc,
                                    const uint8_t* __restrict__ skeys, uint32_t ms, const uint32_t* __restrict__ seg_of_acc, uint32_t n_st,
                                    uint8_t* __restrict__ keys, uint32_t* __restrict__ seg)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na + ms; i += gridDim.x * blockDim.x) {
        if (i < na) { copy32(keys + 32ull * i, akeys + 32ull * i); seg[i] = n_st + ablock[i]; }
        else { copy32(keys + 32ull * i, skeys + 32ull * (i - na)); seg[i] = seg_of_acc[sacc[i - na]]; }
    }
}
// gather in (segment, key) order; flag[0] = some key twice in one segment
__global__ void tr_sorted_keys_kernel(const uint8_t* __restrict__ keys, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ perm, uint32_t n,
                                      uint8_t* __restrict__ skeys, uint32_t* __restrict__ sseg, uint32_t* __restrict__ flag)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t p = perm[i];
        copy32(skeys + 32ull * i, keys + 32ull * p);
        sseg[i] = seg[p];
        if (i && seg[perm[i - 1]] == seg[p] && cmp32(keys + 32ull * perm[i - 1], keys + 32ull * p) == 0) atomicExch(flag, 1u);
    }
}
// off[s] = first index whose segment is >= s, s = 0..n_seg
__global__ void tr_seg_off_kernel(const uint32_t* __restrict__ seg, uint32_t n, uint32_t n_seg, uint32_t* __restrict__ off)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s <= n_seg; s += gridDim.x * blockDim.x) {
        uint32_t a = 0, b = n;
        while (a < b) { const uint32_t mid = (a + b) >> 1; if (seg[mid] < s) a = mid + 1; else b = mid; }
        off[s] = a;
    }
}
__global__ void tr_block_init_kernel(const uint8_t* __restrict__ acc_status, const uint32_t* __restrict__ ablock, uint32_t na, uint32_t* __restrict__ bflags)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        if (acc_status[i] == tn::ST_REJECT) atomicOr(&bflags[ablock[i]], TB_BAD);
        if (acc_status[i] == tn::ST_MISSING) atomicOr(&bflags[ablock[i]], TB_MISSING);
    }
}
// one root per segment of a block the account walk did not fail; an empty trie has nothing to expand
__global__ void tr_front_init_kernel(TSeg g, uint32_t n_seg, const uint32_t* __restrict__ bflags, const uint8_t* __restrict__ pre_roots,
                                     const uint8_t* __restrict__ aflags, const uint8_t* __restrict__ acc_status, const uint8_t* __restrict__ acc_roots,
                                     const uint32_t* __restrict__ key_off, TFront* __restrict__ front, uint32_t* __restrict__ count)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
        const uint32_t b = seg_block(g, s);
        if (bflags[b]) continue;
        const uint8_t* root = pre_roots + 32ull * b;
        if (s < g.n_st) {
            const uint32_t a = g.acc_of_seg[s];
            if ((aflags[a] & PHANT_GPU_ACCOUNT_CLEAR_STORAGE) || acc_status[a] != tn::ST_PRESENT) continue;
            root = acc_roots + 32ull * a;
        }
        bool empty = true;
        for (int i = 0; i < 32; ++i) empty &= root[i] == EMPTY_ROOT_D[i];
        if (empty) continue;
        TFront f{};
        copy32(f.ref, root);
        f.seg = s; f.lo = key_off[s]; f.hi = key_off[s + 1];
        front[atomicAdd(count, 1u)] = f;
    }
}

// One level of the expansion, one node per thread: a hashed node with no diff key under it becomes a stub; otherwise it is
// looked up and decoded -- a leaf becomes a leaf item, an extension or a branch passes each child (and the diff keys under it)
// to the next level.  Embedded children are expanded like any other node.
__global__ void __launch_bounds__(128)
tr_expand_kernel(const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off, const uint8_t* __restrict__ digests, const tn::Bag bag,
                 const uint8_t* __restrict__ keys, const TFront* __restrict__ cur, uint32_t n, TFront* __restrict__ next, TItem* __restrict__ items,
                 uint32_t* __restrict__ counters /*[0] next, [1] items*/, TSeg g, uint32_t* __restrict__ bflags)
{
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const TFront& f = cur[e];
        const uint32_t blk = seg_block(g, f.seg);
        const uint8_t* node;
        uint64_t len;
        if (f.len == 0) {
            if (f.lo == f.hi) {
                TItem& it = items[atomicAdd(&counters[1], 1u)];
                copy32(it.key, f.prefix); copy32(it.ref, f.ref);
                it.voff = 0; it.vlen = 0; it.seg = f.seg; it.depth = f.depth; it.kind = f.below_ext ? TI_STUB_BRANCH : TI_STUB;
                continue;
            }
            uint32_t ex[8];
            tn::load32_aligned(f.ref, ex);
            const uint32_t idx = tn::bag_find(bag, digests, ex);
            if (idx == tn::BAG_EMPTY) { atomicOr(&bflags[blk], TB_MISSING); continue; }
            node = nodes + node_off[idx];
            len = node_off[idx + 1] - node_off[idx];
        } else {
            node = nodes + f.off;
            len = f.len;
        }
        tn::TNode t;
        if (len > 0xffffffffull || !tn::tn_decode(node, (uint32_t)len, t)) { atomicOr(&bflags[blk], TB_BAD); continue; }
        if (t.kind == tn::TN_LEAF) {
            if (f.depth + t.plen != 64) { atomicOr(&bflags[blk], TB_BAD); continue; }
            TItem& it = items[atomicAdd(&counters[1], 1u)];
            copy32(it.key, f.prefix);
            for (uint32_t j = 0; j < t.plen; ++j) tn::tk_set_nibble(it.key, f.depth + j, tn::tn_path_nibble(node, t, j));
            it.voff = (uint64_t)(node + t.val_off - nodes); it.vlen = t.val_len; it.seg = f.seg; it.depth = 64; it.kind = TI_LEAF;
            continue;
        }
        const bool ext = t.kind == tn::TN_EXT;
        const uint32_t step = ext ? t.plen : 1;
        if (ext ? f.depth + step >= 64 : f.depth >= 64) { atomicOr(&bflags[blk], TB_BAD); continue; } // a branch needs a nibble
        for (uint32_t v = 0; v < (ext ? 1u : 16u); ++v) {
            if (t.c_kind[v] == tn::TC_EMPTY) continue;
            uint32_t lo, hi;
            if (ext) tn::tk_ext_range(keys, f.lo, f.hi, f.depth, node, t, lo, hi);
            else { lo = tn::tk_nibble_bound(keys, f.lo, f.hi, f.depth, v); hi = v == 15 ? f.hi : tn::tk_nibble_bound(keys, lo, f.hi, f.depth, v + 1); }
            TFront c;
            copy32(c.prefix, f.prefix);
            if (ext) for (uint32_t j = 0; j < t.plen; ++j) tn::tk_set_nibble(c.prefix, f.depth + j, tn::tn_path_nibble(node, t, j));
            else tn::tk_set_nibble(c.prefix, f.depth, v);
            if (t.c_kind[v] == tn::TC_HASH) { copy32(c.ref, node + t.c_off[v]); c.off = 0; c.len = 0; }
            else { for (int b = 0; b < 32; ++b) c.ref[b] = 0; c.off = (uint64_t)(node + t.c_off[v] - nodes); c.len = t.c_len[v]; }
            c.seg = f.seg; c.depth = f.depth + step; c.lo = lo; c.hi = hi; c.below_ext = ext ? 1 : 0;
            next[atomicAdd(&counters[0], 1u)] = c;
        }
    }
}

// the diff's own items: upserted accounts, written slots, and deletions (which only remove the witness leaf they match)
__global__ void tr_diff_items_kernel(const RsDiff d, const uint32_t* __restrict__ ablock, const uint32_t* __restrict__ seg_of_acc, uint32_t n_st,
                                     TItem* __restrict__ items)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < d.na + d.ms; i += gridDim.x * blockDim.x) {
        TItem& it = items[i];
        it.vlen = 0; it.depth = 64;
        for (int b = 0; b < 32; ++b) it.ref[b] = 0;
        if (i < d.na) {
            copy32(it.key, d.akeys + 32ull * i);
            it.seg = n_st + ablock[i]; it.voff = i;
            it.kind = (d.aflags[i] & PHANT_GPU_ACCOUNT_DELETE) ? TI_DEL : TI_ACC;
        } else {
            const uint32_t j = i - d.na;
            copy32(it.key, d.skeys + 32ull * j);
            it.seg = seg_of_acc[d.sacc[j]]; it.voff = j;
            bool zero = true;
            for (int b = 0; b < 32; ++b) zero &= d.svals[32ull * j + b] == 0;
            it.kind = zero ? TI_DEL : TI_SLOT;
        }
    }
}
__global__ void tr_item_keys_kernel(const TItem* __restrict__ items, uint32_t n, uint8_t* __restrict__ keys, uint32_t* __restrict__ seg)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { copy32(keys + 32ull * i, items[i].key); seg[i] = items[i].seg; }
}
// in (segment, key) order, witness items before diff items of the same key (the sort is stable): a witness leaf the diff lists
// is replaced by it; deletions go; so does every item of a block that has already failed
__global__ void tr_classify_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ perm, uint32_t n, TSeg g, const uint32_t* __restrict__ bflags,
                                   uint32_t* __restrict__ keep)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const TItem& it = items[perm[i]];
        bool k = it.kind != TI_DEL && bflags[seg_block(g, it.seg)] == 0;
        if (k && it.kind == TI_LEAF && i + 1 < n) {
            const TItem& nx = items[perm[i + 1]];
            if (nx.seg == it.seg && cmp32(nx.key, it.key) == 0) k = false;
        }
        keep[i] = k ? 1 : 0;
    }
}
__global__ void tr_compact_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ perm, const uint32_t* __restrict__ keep,
                                  const uint32_t* __restrict__ pos, uint32_t n, uint32_t* __restrict__ cidx, uint8_t* __restrict__ ckeys, uint32_t* __restrict__ cseg)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (!keep[i]) continue;
        const uint32_t p = pos[i], q = perm[i];
        cidx[p] = q;
        copy32(ckeys + 32ull * p, items[q].key);
        cseg[p] = items[q].seg;
    }
}

// The node a stub becomes when the rebuild moves it from its depth up to depth pl: an extension over its reference when it is a
// branch (known without a lookup below an extension), its path lengthened when it is a leaf or an extension.  out == nullptr:
// the size only.  Returns 0 with `flag` set when the node is missing or breaks the rules.
__device__ uint32_t tr_collapsed(const TItem& it, uint32_t pl, const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off,
                                 const uint8_t* __restrict__ digests, const tn::Bag& bag, uint8_t* out, uint32_t& flag)
{
    uint8_t nib[128];
    uint32_t cnt = 0;
    for (uint32_t q = pl; q < it.depth; ++q) nib[cnt++] = (uint8_t)tn::tk_nibble(it.key, q);
    const uint8_t* child = it.ref; // the extension's child: a 32-byte hash, or an embedded node of child_len bytes
    uint32_t child_len = 32;
    bool child_hash = true, leaf = false;
    const uint8_t* val = nullptr;
    uint32_t vlen = 0;
    if (it.kind == TI_STUB) {
        uint32_t ex[8];
        tn::load32_aligned(it.ref, ex);
        const uint32_t idx = tn::bag_find(bag, digests, ex);
        if (idx == tn::BAG_EMPTY) { flag = TB_MISSING; return 0; }
        const uint8_t* node = nodes + node_off[idx];
        const uint64_t len = node_off[idx + 1] - node_off[idx];
        tn::TNode t;
        if (len > 0xffffffffull || !tn::tn_decode(node, (uint32_t)len, t)) { flag = TB_BAD; return 0; }
        if (t.kind != tn::TN_BRANCH) {
            leaf = t.kind == tn::TN_LEAF;
            if (leaf ? it.depth + t.plen != 64 : it.depth + t.plen >= 64) { flag = TB_BAD; return 0; }
            for (uint32_t j = 0; j < t.plen; ++j) nib[cnt++] = (uint8_t)tn::tn_path_nibble(node, t, j);
            if (leaf) { val = node + t.val_off; vlen = t.val_len; }
            else { child = node + t.c_off[0]; child_len = t.c_len[0]; child_hash = t.c_kind[0] == tn::TC_HASH; }
        }
    }
    const uint32_t hpn = 1 + cnt / 2;
    const uint32_t hp0 = ((((leaf ? 2u : 0u) + (cnt & 1)) << 4) | ((cnt & 1) ? nib[0] : 0u));
    const uint32_t s_hp = (uint32_t)str_size(hpn, hp0);
    const uint32_t s_2 = leaf ? (uint32_t)str_size(vlen, vlen ? val[0] : 0) : (child_hash ? 33u : child_len);
    const uint32_t payload = s_hp + s_2, total = hdr_size(payload) + payload;
    if (!out) return total;
    uint8_t* q = out + put_hdr(out, payload, 0xc0, 0xf7);
    if (s_hp > hpn) q += put_hdr(q, hpn, 0x80, 0xb7);
    *q++ = (uint8_t)hp0;
    for (uint32_t j = cnt & 1; j < cnt; j += 2) *q++ = (uint8_t)((nib[j] << 4) | nib[j + 1]);
    if (leaf) {
        if (s_2 > vlen) q += put_hdr(q, vlen, 0x80, 0xb7);
        for (uint32_t b = 0; b < vlen; ++b) *q++ = val[b];
    } else if (child_hash) {
        *q++ = 0xa0;
        for (int b = 0; b < 32; ++b) *q++ = child[b];
    } else {
        for (uint32_t b = 0; b < child_len; ++b) *q++ = child[b];
    }
    return total;
}

// Where each stub hangs after the rebuild: one below the deeper of its two neighbours' common prefixes (0 when it is alone in
// its segment).  At its own depth its reference is cached as it is; higher up it is queued for tr_collapsed.
__global__ void tr_place_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ cidx, const uint8_t* __restrict__ ckeys,
                                const uint32_t* __restrict__ cseg, uint32_t m, const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off,
                                const uint8_t* __restrict__ digests, const tn::Bag bag, TSeg g, uint32_t* __restrict__ bflags, uint8_t* __restrict__ cache,
                                uint32_t* __restrict__ mv_item, uint32_t* __restrict__ mv_pl, uint64_t* __restrict__ mv_size, uint32_t* __restrict__ mv_count)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const TItem& it = items[cidx[i]];
        uint8_t* row = cache + 33ull * i;
        row[0] = 0;
        if (it.kind != TI_STUB && it.kind != TI_STUB_BRANCH) continue;
        uint32_t pl = 0;
        if (i > 0 && cseg[i - 1] == cseg[i]) pl = max(pl, lcp32(ckeys + 32ull * (i - 1), ckeys + 32ull * i) + 1);
        if (i + 1 < m && cseg[i + 1] == cseg[i]) pl = max(pl, lcp32(ckeys + 32ull * (i + 1), ckeys + 32ull * i) + 1);
        const uint32_t blk = seg_block(g, it.seg);
        if (pl > it.depth) { atomicOr(&bflags[blk], TB_BAD); continue; } // cannot happen: no other key lies under a stub's prefix
        if (pl == it.depth) {
            row[0] = (uint8_t)(pl + 1);
            for (int b = 0; b < 32; ++b) row[1 + b] = it.ref[b];
            continue;
        }
        uint32_t flag = 0;
        const uint32_t sz = tr_collapsed(it, pl, nodes, node_off, digests, bag, nullptr, flag);
        if (flag) { atomicOr(&bflags[blk], flag); continue; }
        const uint32_t j = atomicAdd(mv_count, 1u);
        mv_item[j] = i; mv_pl[j] = pl; mv_size[j] = sz;
    }
}
__global__ void tr_collapse_encode_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ cidx, const uint32_t* __restrict__ mv_item,
                                          const uint32_t* __restrict__ mv_pl, uint32_t cnt, const uint64_t* __restrict__ off, uint8_t* __restrict__ arena,
                                          const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off, const uint8_t* __restrict__ digests,
                                          const tn::Bag bag)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        uint32_t flag = 0;
        tr_collapsed(items[cidx[mv_item[j]]], mv_pl[j], nodes, node_off, digests, bag, arena + off[j], flag);
    }
}
// a moved stub's new node is at least as long as the node it was (>= 32 bytes, hence referenced by hash): cache its digest
__global__ void tr_collapse_cache_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ cidx, const uint32_t* __restrict__ mv_item,
                                         const uint32_t* __restrict__ mv_pl, const uint64_t* __restrict__ off, uint32_t cnt, const uint8_t* __restrict__ dg,
                                         TSeg g, uint32_t* __restrict__ bflags, uint8_t* __restrict__ cache)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        const uint32_t i = mv_item[j];
        if (off[j + 1] - off[j] < 32) { atomicOr(&bflags[seg_block(g, items[cidx[i]].seg)], TB_BAD); continue; }
        uint8_t* row = cache + 33ull * i;
        row[0] = (uint8_t)(mv_pl[j] + 1);
        for (int b = 0; b < 32; ++b) row[1 + b] = dg[32ull * j + b];
    }
}

// leaf values for the forest builder: witness leaves as they were, slots as rlp(trim(value)), accounts sized by
// account_size_kernel and written once their storage roots are known; stubs have none
__global__ void tr_val_size_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ cidx, uint32_t m, const uint8_t* __restrict__ svals,
                                   const uint64_t* __restrict__ asize, uint64_t* __restrict__ size)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const TItem& it = items[cidx[i]];
        uint64_t sz = 0;
        if (it.kind == TI_LEAF) sz = it.vlen;
        else if (it.kind == TI_ACC) sz = asize[it.voff];
        else if (it.kind == TI_SLOT) {
            const uint8_t* v = svals + 32ull * it.voff;
            uint32_t z = 0;
            while (z < 32 && v[z] == 0) ++z;
            sz = str_size(32 - z, v[z]);
        }
        size[i] = sz;
    }
}
__global__ void tr_val_fill_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ cidx, uint32_t m, const uint8_t* __restrict__ nodes,
                                   const uint8_t* __restrict__ svals, const uint64_t* __restrict__ voff, uint8_t* __restrict__ arena, uint32_t* __restrict__ key_off)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= m; i += gridDim.x * blockDim.x) {
        key_off[i] = 32u * i;
        if (i == m) break;
        const TItem& it = items[cidx[i]];
        uint8_t* out = arena + voff[i];
        if (it.kind == TI_LEAF) {
            for (uint32_t b = 0; b < it.vlen; ++b) out[b] = nodes[it.voff + b];
        } else if (it.kind == TI_SLOT) {
            const uint8_t* v = svals + 32ull * it.voff;
            uint32_t z = 0;
            while (z < 32 && v[z] == 0) ++z;
            if (voff[i + 1] - voff[i] > 32 - z) *out++ = (uint8_t)(0x80 + 32 - z);
            for (uint32_t b = z; b < 32; ++b) *out++ = v[b];
        }
    }
}
__global__ void tr_acc_vals_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ cidx, uint32_t m, const uint64_t* __restrict__ body_off,
                                   const uint8_t* __restrict__ bodies, const uint64_t* __restrict__ voff, uint8_t* __restrict__ arena)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const TItem& it = items[cidx[i]];
        if (it.kind != TI_ACC) continue;
        const uint64_t a = it.voff;
        for (uint64_t b = 0; b < body_off[a + 1] - body_off[a]; ++b) arena[voff[i] + b] = bodies[body_off[a] + b];
    }
}
// each listed account's storage root: its storage segment's root (zero for DELETE accounts, which have none)
__global__ void tr_sroot_kernel(const uint8_t* __restrict__ aflags, uint32_t na, const uint32_t* __restrict__ seg_of_acc, const uint8_t* __restrict__ st_roots,
                                uint8_t* __restrict__ sroot)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        const bool del = aflags[i] & PHANT_GPU_ACCOUNT_DELETE;
        for (int b = 0; b < 32; ++b) sroot[32ull * i + b] = del ? 0 : st_roots[32ull * seg_of_acc[i] + b];
    }
}
__global__ void tr_rebase_kernel(const uint32_t* __restrict__ in, uint32_t n, uint32_t base, uint32_t* __restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = in[i] - base;
}
// outputs: status per block, roots only where it is 1
__global__ void tr_out_kernel(const uint32_t* __restrict__ bflags, uint32_t nb, const uint8_t* __restrict__ acc_roots, const uint32_t* __restrict__ ablock,
                              uint32_t na, uint8_t* __restrict__ sroot, uint8_t* __restrict__ post, uint8_t* __restrict__ status)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nb + na; i += gridDim.x * blockDim.x) {
        if (i < nb) {
            const uint32_t f = bflags[i];
            const uint8_t st = (f & TB_BAD) ? tn::ST_REJECT : (f & TB_MISSING) ? tn::ST_MISSING : 1;
            status[i] = st;
            for (int b = 0; b < 32; ++b) post[32ull * i + b] = st == 1 ? acc_roots[32ull * i + b] : 0;
        } else if (bflags[ablock[i - nb]]) {
            for (int b = 0; b < 32; ++b) sroot[32ull * (i - nb) + b] = 0;
        }
    }
}

// grow a device buffer to `need` bytes keeping its first `used` bytes
int grow_keep(phant_gpu_ctx* ctx, DevBuf& b, uint64_t used, uint64_t need)
{
    if (need <= b.cap) return PHANT_GPU_OK;
    DevBuf nb;
    RC(nb.reserve(ctx, need + need / 2));
    if (used) CU(cudaMemcpyAsync(nb.ptr, b.ptr, used, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    b.release();
    b = nb;
    return PHANT_GPU_OK;
}

int read_u32(phant_gpu_ctx* ctx, const uint32_t* d, uint32_t* h, uint32_t n = 1)
{
    CU(cudaMemcpyAsync(h, d, 4ull * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return PHANT_GPU_OK;
}

// ---- the stub-rebuild pipeline's shared steps, in the order T and G run them ----

// Expand the n_front nodes in tr_front[0] one level per launch along the sorted `keys`, appending items to tr_items from
// index first_item (counters[1] must already hold it); tr_items keeps room for `extra` more items behind them.
int tr_expand_all(phant_gpu_ctx* ctx, const uint8_t* nodes, const uint64_t* node_off, const uint8_t* digests, const tn::Bag& bag,
                  const uint8_t* keys, const TSeg& g, uint32_t* bflags, uint32_t* counters, uint32_t n_front, uint32_t first_item,
                  uint32_t extra, uint32_t& n_items)
{
    cudaStream_t s = ctx->stream;
    uint32_t cur_n = n_front, levels = 0;
    n_items = first_item;
    int cur = 0;
    while (cur_n) {
        if (++levels > 70) return PHANT_GPU_E_CUDA; // cannot happen: every level consumes at least one of the 64 nibbles
        RC(ctx->tr_front[1 - cur].reserve(ctx, sizeof(TFront) * 16ull * cur_n));
        RC(grow_keep(ctx, ctx->tr_items, sizeof(TItem) * (uint64_t)n_items, sizeof(TItem) * ((uint64_t)n_items + cur_n + extra + 1)));
        CU(cudaMemsetAsync(counters, 0, 4, s));
        tr_expand_kernel<<<grid1d(ctx->device, cur_n, 128), 128, 0, s>>>(nodes, node_off, digests, bag, keys, (const TFront*)ctx->tr_front[cur].ptr,
                                                                         cur_n, (TFront*)ctx->tr_front[1 - cur].ptr, (TItem*)ctx->tr_items.ptr,
                                                                         counters, g, bflags);
        ctx->stats.launches++;
        uint32_t h[2];
        RC(read_u32(ctx, counters, h, 2));
        cur_n = h[0];
        n_items = h[1];
        cur = 1 - cur;
    }
    return PHANT_GPU_OK;
}

// tr_work's shared prefix for n items in n_seg segments; each caller carves its own arrays behind it in the same carve
struct TrWork {
    uint8_t *ikeys, *ckeys, *cache;
    uint32_t *iseg, *iperm, *keep, *pos, *cidx, *cseg, *mv_item, *mv_pl, *key_off, *seg_off;
    uint64_t *mv_size, *mv_off, *voff;
    uint32_t n, n_seg;
    void take(Carve& c, uint32_t n_items, uint32_t n_segs)
    {
        n = n_items;
        n_seg = n_segs;
        ikeys = c.take<uint8_t>(32ull * n); iseg = c.take<uint32_t>(n); iperm = c.take<uint32_t>(n);
        keep = c.take<uint32_t>(n + 1); pos = c.take<uint32_t>(n + 1);
        cidx = c.take<uint32_t>(n); ckeys = c.take<uint8_t>(32ull * n); cseg = c.take<uint32_t>(n); cache = c.take<uint8_t>(33ull * n);
        mv_item = c.take<uint32_t>(n); mv_pl = c.take<uint32_t>(n); mv_size = c.take<uint64_t>(n + 1); mv_off = c.take<uint64_t>(n + 1);
        voff = c.take<uint64_t>(n + 1); key_off = c.take<uint32_t>(n + 1); seg_off = c.take<uint32_t>(n_seg + 1);
    }
};

// Sort the items by (segment, key), mark in w.keep which to keep (`classify` launches the one kernel that writes
// w.keep[0, n) in sorted order) and compact them into w.cidx / w.ckeys / w.cseg; m = how many were kept.
template <class Classify> int tr_sort_keep(phant_gpu_ctx* ctx, const TItem* items, const TrWork& w, Classify&& classify, uint32_t& m)
{
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t n = w.n;
    m = 0;
    if (!n) return PHANT_GPU_OK;
    tr_item_keys_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(items, n, w.ikeys, w.iseg);
    ctx->stats.launches++;
    RC(sort_by_segment_and_hash(ctx, w.ikeys, w.iseg, n, w.iperm, ctx->tr_sort));
    classify();
    CU(cudaMemsetAsync(w.keep + n, 0, 4, s));
    RC(scan_u32(ctx, w.keep, w.pos, n + 1));
    tr_compact_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(items, w.iperm, w.keep, w.pos, n, w.cidx, w.ckeys, w.cseg);
    ctx->stats.launches += 3;
    return read_u32(ctx, w.pos + n, &m);
}

// Where each of the m kept stubs hangs (w.cache); the nodes of the stubs the rebuild moves up, encoded into tr_vals and hashed
int tr_place_stubs(phant_gpu_ctx* ctx, const TItem* items, const TrWork& w, uint32_t m, const uint8_t* nodes, const uint64_t* node_off,
                   const uint8_t* digests, const tn::Bag& bag, const TSeg& g, uint32_t* bflags, uint32_t* counters)
{
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    if (!m) return PHANT_GPU_OK;
    tr_place_kernel<<<grid1d(dev, m, 128), 128, 0, s>>>(items, w.cidx, w.ckeys, w.cseg, m, nodes, node_off, digests, bag, g, bflags, w.cache,
                                                        w.mv_item, w.mv_pl, w.mv_size, counters + 2);
    ctx->stats.launches++;
    uint32_t mv = 0;
    RC(read_u32(ctx, counters + 2, &mv));
    if (!mv) return PHANT_GPU_OK;
    RC(scan_sizes(ctx, w.mv_size, w.mv_off, mv));
    uint64_t total = 0;
    CU(cudaMemcpyAsync(&total, w.mv_off + mv, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    uint8_t *arena, *dg;
    RC(carve(ctx, ctx->tr_vals, [&](Carve& c) { arena = c.take<uint8_t>(total + 64); dg = c.take<uint8_t>(32ull * mv); }));
    tr_collapse_encode_kernel<<<grid1d(dev, mv, 128), 128, 0, s>>>(items, w.cidx, w.mv_item, w.mv_pl, mv, w.mv_off, arena, nodes, node_off, digests, bag);
    RC(ctx->hash_csr(arena, w.mv_off, mv, total, dg));
    tr_collapse_cache_kernel<<<grid1d(dev, mv, 256), 256, 0, s>>>(items, w.cidx, w.mv_item, w.mv_pl, w.mv_off, mv, dg, g, bflags, w.cache);
    ctx->stats.launches += 3;
    return PHANT_GPU_OK;
}

// The m kept items' leaf values in one tr_vals arena at w.voff, with w.key_off and w.seg_off for build_forest.  T passes its
// slot values, account sizes and, on the device, the size of the account-body area carved behind the arena (read back after
// the values' size); G passes null for all three.
int tr_values(phant_gpu_ctx* ctx, const TItem* items, const TrWork& w, uint32_t m, const uint8_t* nodes, const uint8_t* svals,
              const uint64_t* asize, const uint64_t* d_bodies_size, uint8_t*& arena, uint8_t*& bodies)
{
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    uint64_t vtotal = 0;
    if (m) {
        tr_val_size_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(items, w.cidx, m, svals, asize, w.mv_size);
        ctx->stats.launches++;
        RC(scan_sizes(ctx, w.mv_size, w.voff, m));
        CU(cudaMemcpyAsync(&vtotal, w.voff + m, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    uint64_t btotal = 0;
    if (d_bodies_size) {
        CU(cudaMemcpyAsync(&btotal, d_bodies_size, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    RC(carve(ctx, ctx->tr_vals, [&](Carve& c) { arena = c.take<uint8_t>(vtotal); bodies = c.take<uint8_t>(btotal); }));
    tr_val_fill_kernel<<<grid1d(dev, m + 1, 256), 256, 0, s>>>(items, w.cidx, m, nodes, svals, w.voff, arena, w.key_off);
    tr_seg_off_kernel<<<grid1d(dev, w.n_seg + 1, 256), 256, 0, s>>>(w.cseg, m, w.n_seg, w.seg_off);
    ctx->stats.launches += 2;
    return PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_transition_roots(phant_gpu_ctx* ctx, const phant_gpu_transition* in, const phant_gpu_state_diff* diff,
                                          uint8_t* post_roots32, uint8_t* status, uint8_t* storage_roots32)
{
    if (!ctx || !in || !diff || !post_roots32 || !status) return PHANT_GPU_E_INVALID;
    // ---- host-side checks: nothing is launched, nothing written, on a bad argument ----
    RC(check_diff_host(ctx, diff));
    const uint64_t nb64 = in->n_blocks, nn = in->n_nodes;
    if (nb64 == 0 || nb64 >= (1ull << 28) || !in->pre_roots32 || nn > (1ull << 30) || (nn && !in->node_off)) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({in->nodes, in->node_off, in->pre_roots32, in->account_block, post_roots32, status, storage_roots32})) return PHANT_GPU_E_INVALID;
    const uint32_t nb = (uint32_t)nb64, na = (uint32_t)diff->n_accounts, ms = (uint32_t)diff->n_slots;
    uint64_t nodes_total = 0;
    if (nn) RC(check_offsets_host(in->node_off, nn, &nodes_total));
    if (nodes_total && !in->nodes) return PHANT_GPU_E_INVALID;
    std::vector<uint32_t> ablock(na ? na : 1, 0), seg_of_acc(na ? na : 1, NONE), acc_of_seg;
    for (uint32_t i = 0; i < na; ++i) {
        if (in->account_block) { if (in->account_block[i] >= nb) return PHANT_GPU_E_INVALID; ablock[i] = in->account_block[i]; }
        if (!(diff->account_flags && (diff->account_flags[i] & PHANT_GPU_ACCOUNT_DELETE))) {
            seg_of_acc[i] = (uint32_t)acc_of_seg.size();
            acc_of_seg.push_back(i);
        }
    }
    const uint32_t n_st = (uint32_t)acc_of_seg.size(), n_seg = n_st + nb, nd = na + ms;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;

    // ---- stage: the diff, then per account its block, segment and walk root; per segment its account; the pre-roots ----
    std::vector<uint8_t> aroots(32ull * (na ? na : 1));
    for (uint32_t i = 0; i < na; ++i) memcpy(&aroots[32ull * i], in->pre_roots32 + 32ull * ablock[i], 32);
    RsDiff dd;
    uint32_t *d_ablock, *d_segacc, *d_accseg;
    uint8_t *d_aroots, *d_pre;
    RC(carve(ctx, ctx->tr_in, [&](Carve& c) {
        dd.take(c, na, ms);
        d_ablock = c.take<uint32_t>(na); d_segacc = c.take<uint32_t>(na); d_accseg = c.take<uint32_t>(n_st);
        d_aroots = c.take<uint8_t>(32ull * na); d_pre = c.take<uint8_t>(32ull * nb);
    }));
    RC(stage_diff(ctx, diff, dd));
    if (na) {
        CU(cudaMemcpyAsync(d_ablock, ablock.data(), 4ull * na, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(d_segacc, seg_of_acc.data(), 4ull * na, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(d_aroots, aroots.data(), 32ull * na, cudaMemcpyHostToDevice, s));
    }
    if (n_st) CU(cudaMemcpyAsync(d_accseg, acc_of_seg.data(), 4ull * n_st, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_pre, in->pre_roots32, 32ull * nb, cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += 40ull * na + 4ull * na + 4ull * n_st + 32ull * nb;
    RC(ctx->upload_csr(in->nodes, in->node_off, nn, nodes_total, 0));
    const uint8_t* d_nodes = (const uint8_t*)ctx->d_msgs.ptr;
    const uint64_t* d_noff = (const uint64_t*)ctx->d_off.ptr;
    const TSeg g{n_st, d_accseg, d_ablock};

    // ---- the diff keys in (segment, key) order; a key twice in one segment is refused before anything is written ----
    uint8_t *dkeys, *skeys, *rec, *sroot, *akeys_scratch;
    uint32_t *dseg, *dperm, *sseg, *key_lo, *counters, *bflags, *akoff_scratch, *acc_iota;
    uint64_t *asize, *body_off;
    RC(carve(ctx, ctx->tr_keys, [&](Carve& c) {
        dkeys = c.take<uint8_t>(32ull * nd); dseg = c.take<uint32_t>(nd); dperm = c.take<uint32_t>(nd);
        skeys = c.take<uint8_t>(32ull * nd); sseg = c.take<uint32_t>(nd);
        key_lo = c.take<uint32_t>(n_seg + 1); counters = c.take<uint32_t>(16); bflags = c.take<uint32_t>(nb);
        rec = c.take<uint8_t>(33ull * na); // account walk: storage roots (32 * na), then status bytes
        sroot = c.take<uint8_t>(32ull * na); asize = c.take<uint64_t>(na + 1); body_off = c.take<uint64_t>(na + 1);
        akeys_scratch = c.take<uint8_t>(32ull * na); akoff_scratch = c.take<uint32_t>(na + 1); acc_iota = c.take<uint32_t>(na + 1);
    }));
    CU(cudaMemsetAsync(counters, 0, 64, s));
    CU(cudaMemsetAsync(bflags, 0, 4ull * nb, s));
    if (nd) {
        tr_diff_keys_kernel<<<grid1d(dev, nd, 256), 256, 0, s>>>(dd.akeys, d_ablock, na, dd.sacc, dd.skeys, ms, d_segacc, n_st, dkeys, dseg);
        ctx->stats.launches++;
        RC(sort_by_segment_and_hash(ctx, dkeys, dseg, nd, dperm, ctx->tr_sort));
        tr_sorted_keys_kernel<<<grid1d(dev, nd, 256), 256, 0, s>>>(dkeys, dseg, dperm, nd, skeys, sseg, counters + 15);
        ctx->stats.launches++;
        uint32_t dup = 0;
        RC(read_u32(ctx, counters + 15, &dup));
        if (dup) return PHANT_GPU_E_INVALID;
    }
    tr_seg_off_kernel<<<grid1d(dev, n_seg + 1, 256), 256, 0, s>>>(sseg, nd, n_seg, key_lo);
    ctx->stats.launches++;

    // ---- the node set, hashed once into W's digest table; the account walk from each block's root (P) ----
    NodeTable t;
    RC(ctx->node_table(d_nodes, d_noff, nn, nodes_total, true, &t));
    const tn::Bag bag{t.table, t.capacity - 1};
    uint8_t* acc_roots = rec;
    uint8_t* acc_status = rec + 32ull * na;
    if (na) {
        CU(launch_read_accounts(s, dev, na, d_nodes, d_noff, t.digests, t.summary, t.table, t.capacity, dd.akeys, d_aroots, na, nullptr, nullptr, 0,
                                acc_roots, acc_status, StateOut{}));
        tr_block_init_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(acc_status, d_ablock, na, bflags);
        ctx->stats.launches += 2;
    }

    // ---- expand the paths of the listed keys, one level per launch ----
    RC(ctx->tr_front[0].reserve(ctx, sizeof(TFront) * (n_seg + 1)));
    tr_front_init_kernel<<<grid1d(dev, n_seg, 256), 256, 0, s>>>(g, n_seg, bflags, d_pre, dd.aflags, acc_status, acc_roots, key_lo,
                                                                 (TFront*)ctx->tr_front[0].ptr, counters);
    ctx->stats.launches++;
    uint32_t h[2] = {0, 0}, n_items = 0;
    RC(read_u32(ctx, counters, h, 2));
    RC(tr_expand_all(ctx, d_nodes, d_noff, t.digests, bag, skeys, g, bflags, counters, h[0], 0, nd, n_items));

    // ---- the diff's items beside the witness's; sort; replace, delete, drop failed blocks ----
    RC(grow_keep(ctx, ctx->tr_items, sizeof(TItem) * (uint64_t)n_items, sizeof(TItem) * ((uint64_t)n_items + nd + 1)));
    TItem* items = (TItem*)ctx->tr_items.ptr;
    if (nd) {
        tr_diff_items_kernel<<<grid1d(dev, nd, 256), 256, 0, s>>>(dd, d_ablock, d_segacc, n_st, items + n_items);
        ctx->stats.launches++;
    }
    TrWork w;
    uint8_t *st_roots, *acc_out;
    uint32_t* acc_seg_off;
    RC(carve(ctx, ctx->tr_work, [&](Carve& c) {
        w.take(c, n_items + nd, n_seg);
        acc_seg_off = c.take<uint32_t>(nb + 1); st_roots = c.take<uint8_t>(32ull * (n_st + 1)); acc_out = c.take<uint8_t>(32ull * nb);
    }));
    uint32_t m = 0;
    RC(tr_sort_keep(ctx, items, w, [&] { tr_classify_kernel<<<grid1d(dev, w.n, 256), 256, 0, s>>>(items, w.iperm, w.n, g, bflags, w.keep); }, m));

    // ---- where each stub hangs; the nodes of the stubs the rebuild moves up ----
    RC(tr_place_stubs(ctx, items, w, m, d_nodes, d_noff, t.digests, bag, g, bflags, counters));

    // ---- leaf values; the storage forest; account bodies with the new storage roots; the account forest ----
    if (na) {
        iota_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(acc_iota, na);
        account_size_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(dd.nonce, dd.bal, acc_iota, na, asize);
        ctx->stats.launches += 2;
        RC(scan_sizes(ctx, asize, body_off, na));
    }
    uint8_t *arena, *bodies;
    RC(tr_values(ctx, items, w, m, d_nodes, dd.svals, asize, na ? body_off + na : nullptr, arena, bodies));
    uint32_t m_st = 0;
    RC(read_u32(ctx, w.seg_off + n_st, &m_st));
    if (n_st) RC(build_forest(ctx, {.keys = w.ckeys, .key_off = w.key_off, .vals = arena, .val_off = w.voff, .n = m_st, .seg_off = w.seg_off,
                                    .n_seg = n_st, .seg_of_key = w.cseg, .roots = st_roots, .leaf_cache = w.cache}));
    if (na) {
        tr_sroot_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(dd.aflags, na, d_segacc, st_roots, sroot);
        account_fill_kernel<<<grid1d(dev, na + 1, 256), 256, 0, s>>>(dd.nonce, dd.bal, sroot, dd.code, dd.akeys, acc_iota, na, body_off, akeys_scratch,
                                                                   akoff_scratch, bodies);
        ctx->stats.launches += 2;
        if (m) {
            tr_acc_vals_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(items, w.cidx, m, body_off, bodies, w.voff, arena);
            ctx->stats.launches++;
        }
    }
    tr_rebase_kernel<<<grid1d(dev, nb + 1, 256), 256, 0, s>>>(w.seg_off + n_st, nb + 1, m_st, acc_seg_off);
    ctx->stats.launches++;
    RC(build_forest(ctx, {.keys = w.ckeys, .key_off = w.key_off + m_st, .vals = arena, .val_off = w.voff + m_st, .n = m - m_st, .seg_off = acc_seg_off,
                          .n_seg = nb, .seg_of_key = w.cseg + m_st, .roots = acc_out, .leaf_cache = w.cache + 33ull * m_st}));

    // ---- outputs (the sort scratch is free by now) ----
    uint8_t *o_post, *o_status;
    RC(carve(ctx, ctx->tr_sort, [&](Carve& c) { o_post = c.take<uint8_t>(32ull * nb); o_status = c.take<uint8_t>(nb); }));
    tr_out_kernel<<<grid1d(dev, nb + na, 256), 256, 0, s>>>(bflags, nb, acc_out, d_ablock, na, sroot, o_post, o_status);
    ctx->stats.launches++;
    CU(cudaMemcpyAsync(post_roots32, o_post, 32ull * nb, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(status, o_status, nb, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += 33ull * nb;
    if (storage_roots32 && na) {
        CU(cudaMemcpyAsync(storage_roots32, sroot, 32ull * na, cudaMemcpyDeviceToHost, s));
        ctx->stats.d2h_bytes += 32ull * na;
    }
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// G: range proofs (include/phant_gpu.h, DESIGN.md §4.3j).  T's pipeline with one segment per range (TSeg with n_st = 0, so a
// segment's flags are its range's): the boundary proofs are expanded along each range's two edge keys, the entries join the
// proof's items as leaves whose values sit right behind the node bytes, a proof item inside [origin, last] is dropped in
// favour of the entries (range_proof.cuh), and each range's forest root is compared with its claimed root.
// ------------------------------------------------------------------------------------------------
namespace rs_body {
#include "range_proof.cuh"
}
namespace rp = rs_body::phant;
namespace {

// one thread per entry: its range, the entry checks, and its leaf item (items[i]; the value at nodes + vbase + val_off[i])
__global__ void rp_entry_kernel(const uint8_t* __restrict__ keys, const uint64_t* __restrict__ val_off, uint64_t vbase,
                                const uint64_t* __restrict__ first, uint32_t nr, uint32_t ne, const uint8_t* __restrict__ flags,
                                const uint8_t* __restrict__ origins, TItem* __restrict__ items, uint32_t* __restrict__ bflags)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ne; i += gridDim.x * blockDim.x) {
        uint32_t a = 0, b = nr; // the last range r with first[r] <= i
        while (b - a > 1) { const uint32_t mid = (a + b) >> 1; if (first[mid] <= i) a = mid; else b = mid; }
        const uint8_t* key = keys + 32ull * i;
        const uint64_t vlen = val_off[i + 1] - val_off[i];
        const bool whole = flags && (flags[a] & PHANT_GPU_RANGE_WHOLE);
        if (!rp::rp_entry_ok(key, i > first[a] ? key - 32 : nullptr, origins + 32ull * a, whole, vlen)) atomicOr(&bflags[a], TB_BAD);
        TItem& it = items[i];
        copy32(it.key, key);
        for (int k = 0; k < 32; ++k) it.ref[k] = 0;
        it.voff = vbase + val_off[i]; it.vlen = (uint32_t)vlen; it.seg = a; it.depth = 64; it.kind = TI_LEAF;
    }
}
// per range: its edge keys (edges[2r] = origin, edges[2r + 1] = last) and, unless it is WHOLE, has failed its entry checks or
// claims the empty root, its root as the first node to expand, with one edge key under it when origin == last, else two
__global__ void rp_front_init_kernel(uint32_t nr, const uint8_t* __restrict__ roots, const uint8_t* __restrict__ origins,
                                     const uint8_t* __restrict__ flags, const uint64_t* __restrict__ first, const uint8_t* __restrict__ keys,
                                     const uint32_t* __restrict__ bflags, uint8_t* __restrict__ edges, TFront* __restrict__ front,
                                     uint32_t* __restrict__ count)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < nr; r += gridDim.x * blockDim.x) {
        uint8_t* o = edges + 64ull * r;
        copy32(o, origins + 32ull * r);
        rp::rp_last(first[r + 1] > first[r] ? keys + 32ull * (first[r + 1] - 1) : nullptr, o + 32);
        if ((flags && (flags[r] & PHANT_GPU_RANGE_WHOLE)) || bflags[r]) continue;
        const uint8_t* root = roots + 32ull * r;
        bool empty = true;
        for (int i = 0; i < 32; ++i) empty &= root[i] == EMPTY_ROOT_D[i];
        if (empty) continue;
        TFront f{};
        copy32(f.ref, root);
        f.seg = r; f.lo = 2 * r; f.hi = 2 * r + (cmp32(o, o + 32) == 0 ? 1 : 2);
        front[atomicAdd(count, 1u)] = f;
    }
}
// in (range, key) order: the entries (items [0, n_entries)) stay; a proof item inside [origin, last] goes, one outside stays
// and sets `more` when it lies above `last`; every item of a range that has already failed goes
__global__ void rp_classify_kernel(const TItem* __restrict__ items, const uint32_t* __restrict__ perm, uint32_t n, uint32_t ne,
                                   const uint8_t* __restrict__ edges, const uint32_t* __restrict__ bflags, uint32_t* __restrict__ keep,
                                   uint32_t* __restrict__ more)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t q = perm[i];
        const TItem& it = items[q];
        bool k = bflags[it.seg] == 0;
        if (k && q >= ne) {
            const uint8_t* o = edges + 64ull * it.seg;
            if (rp::rp_inside(it.key, it.kind == TI_LEAF ? 64u : it.depth, o, o + 32)) k = false;
            else if (rp::rp_above(it.key, o + 32)) more[it.seg] = 1;
        }
        keep[i] = k ? 1 : 0;
    }
}
__global__ void rp_out_kernel(const uint32_t* __restrict__ bflags, uint32_t nr, const uint8_t* __restrict__ built, const uint8_t* __restrict__ roots,
                              const uint32_t* __restrict__ more_flag, uint8_t* __restrict__ status, uint8_t* __restrict__ more)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < nr; r += gridDim.x * blockDim.x) {
        const uint32_t f = bflags[r];
        uint8_t st = (f & TB_BAD) ? tn::ST_REJECT : (f & TB_MISSING) ? tn::ST_MISSING : 1;
        if (st == 1 && cmp32(built + 32ull * r, roots + 32ull * r) != 0) st = tn::ST_REJECT;
        status[r] = st;
        more[r] = st == 1 && more_flag[r] ? 1 : 0;
    }
}

} // namespace

extern "C" int phant_gpu_verify_ranges(phant_gpu_ctx* ctx, const phant_gpu_range_proofs* in, uint8_t* status, uint8_t* more)
{
    if (!ctx || !in) return PHANT_GPU_E_INVALID;
    // ---- host-side checks: nothing is launched, nothing written, on a bad argument ----
    const uint64_t nr64 = in->n_ranges, nn = in->n_nodes;
    if (nr64 == 0) return PHANT_GPU_OK;
    if (!status || !in->roots32 || !in->origin32 || !in->entry_first || nr64 > (1ull << 30) || nn > (1ull << 30) || (nn && !in->node_off))
        return PHANT_GPU_E_INVALID;
    if (!host_ptrs({in->nodes, in->node_off, in->roots32, in->origin32, in->range_flags, in->entry_first, in->keys32, in->vals, in->val_off,
                    status, more}))
        return PHANT_GPU_E_INVALID;
    const uint32_t nr = (uint32_t)nr64;
    if (in->entry_first[0] != 0) return PHANT_GPU_E_INVALID;
    for (uint32_t r = 0; r < nr; ++r) {
        if (in->entry_first[r + 1] < in->entry_first[r]) return PHANT_GPU_E_INVALID;
        if (in->range_flags && (in->range_flags[r] & ~PHANT_GPU_RANGE_WHOLE)) return PHANT_GPU_E_INVALID;
    }
    const uint64_t ne64 = in->entry_first[nr];
    if (ne64 > (1ull << 30) || (ne64 && (!in->keys32 || !in->val_off))) return PHANT_GPU_E_INVALID;
    const uint32_t ne = (uint32_t)ne64;
    uint64_t nodes_total = 0, vals_total = 0;
    if (nn) RC(check_offsets_host(in->node_off, nn, &nodes_total));
    if (ne) {
        for (uint32_t i = 0; i < ne; ++i)
            if (in->val_off[i + 1] < in->val_off[i] || in->val_off[i + 1] - in->val_off[i] > 0xffffffffull) return PHANT_GPU_E_INVALID;
        vals_total = in->val_off[ne];
    }
    if ((nodes_total && !in->nodes) || (vals_total && !in->vals)) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;

    // ---- stage: the node set with the entry values behind it; per range its root, origin, flags and entry CSR; the entries ----
    uint8_t *d_roots, *d_origins, *d_flags, *d_keys, *edges;
    uint64_t *d_first, *d_voff;
    uint32_t *counters, *bflags, *more_flag;
    RC(carve(ctx, ctx->tr_in, [&](Carve& c) {
        d_roots = c.take<uint8_t>(32ull * nr); d_origins = c.take<uint8_t>(32ull * nr); d_flags = c.take<uint8_t>(nr);
        d_first = c.take<uint64_t>(nr + 1); d_keys = c.take<uint8_t>(32ull * ne); d_voff = c.take<uint64_t>(ne + 1);
        edges = c.take<uint8_t>(64ull * nr); counters = c.take<uint32_t>(16); bflags = c.take<uint32_t>(nr); more_flag = c.take<uint32_t>(nr);
    }));
    RC(ctx->upload_csr(in->nodes, in->node_off, nn, nodes_total, vals_total));
    const uint8_t* d_nodes = (const uint8_t*)ctx->d_msgs.ptr;
    if (vals_total) CU(cudaMemcpyAsync((uint8_t*)ctx->d_msgs.ptr + nodes_total, in->vals, vals_total, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_roots, in->roots32, 32ull * nr, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_origins, in->origin32, 32ull * nr, cudaMemcpyHostToDevice, s));
    if (in->range_flags) CU(cudaMemcpyAsync(d_flags, in->range_flags, nr, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_first, in->entry_first, 8ull * (nr + 1), cudaMemcpyHostToDevice, s));
    if (ne) {
        CU(cudaMemcpyAsync(d_keys, in->keys32, 32ull * ne, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(d_voff, in->val_off, 8ull * (ne + 1), cudaMemcpyHostToDevice, s));
    }
    ctx->stats.h2d_bytes += vals_total + 64ull * nr + (in->range_flags ? nr : 0) + 8ull * (nr + 1) +
                            (ne ? 32ull * ne + 8ull * (ne + 1) : 0);
    const uint64_t* d_noff = (const uint64_t*)ctx->d_off.ptr;
    const uint8_t* d_fl = in->range_flags ? d_flags : nullptr;
    const TSeg g{0, nullptr, nullptr};
    CU(cudaMemsetAsync(counters, 0, 64, s));
    CU(cudaMemsetAsync(bflags, 0, 4ull * nr, s));
    CU(cudaMemsetAsync(more_flag, 0, 4ull * nr, s));

    // ---- the node set, hashed once into W's digest table (no walk here: no summaries) ----
    NodeTable t;
    RC(ctx->node_table(d_nodes, d_noff, nn, nodes_total, false, &t));
    const tn::Bag bag{t.table, t.capacity - 1};

    // ---- the entries: checks and leaf items (items [0, ne)); each range's edge keys and root ----
    RC(grow_keep(ctx, ctx->tr_items, 0, sizeof(TItem) * ((uint64_t)ne + 1)));
    if (ne) {
        rp_entry_kernel<<<grid1d(dev, ne, 256), 256, 0, s>>>(d_keys, d_voff, nodes_total, d_first, nr, ne, d_fl, d_origins, (TItem*)ctx->tr_items.ptr,
                                                             bflags);
        ctx->stats.launches++;
    }
    RC(ctx->tr_front[0].reserve(ctx, sizeof(TFront) * (nr + 1)));
    rp_front_init_kernel<<<grid1d(dev, nr, 256), 256, 0, s>>>(nr, d_roots, d_origins, d_fl, d_first, d_keys, bflags, edges,
                                                              (TFront*)ctx->tr_front[0].ptr, counters);
    ctx->stats.launches++;

    // ---- expand the boundary proofs along the edge keys, one level per launch, behind the entries ----
    uint32_t h[2] = {0, 0}, n_items = ne;
    RC(read_u32(ctx, counters, h, 2));
    CU(cudaMemcpyAsync(counters + 1, &n_items, 4, cudaMemcpyHostToDevice, s));
    RC(tr_expand_all(ctx, d_nodes, d_noff, t.digests, bag, edges, g, bflags, counters, h[0], ne, 0, n_items));

    // ---- sort the entries and the proof's items together; drop what lies inside each range ----
    TItem* items = (TItem*)ctx->tr_items.ptr;
    TrWork w;
    uint8_t *built, *o_status, *o_more;
    RC(carve(ctx, ctx->tr_work, [&](Carve& c) {
        w.take(c, n_items, nr);
        built = c.take<uint8_t>(32ull * nr); o_status = c.take<uint8_t>(nr); o_more = c.take<uint8_t>(nr);
    }));
    uint32_t m = 0;
    RC(tr_sort_keep(ctx, items, w, [&] {
        rp_classify_kernel<<<grid1d(dev, w.n, 256), 256, 0, s>>>(items, w.iperm, w.n, ne, edges, bflags, w.keep, more_flag);
    }, m));

    // ---- where each stub hangs; the nodes of the stubs the rebuild moves up ----
    RC(tr_place_stubs(ctx, items, w, m, d_nodes, d_noff, t.digests, bag, g, bflags, counters));

    // ---- leaf values (proof leaves and entries alike sit in the node buffer); one forest of every range's trie ----
    uint8_t *arena, *no_bodies;
    RC(tr_values(ctx, items, w, m, d_nodes, nullptr, nullptr, nullptr, arena, no_bodies));
    RC(build_forest(ctx, {.keys = w.ckeys, .key_off = w.key_off, .vals = arena, .val_off = w.voff, .n = m, .seg_off = w.seg_off, .n_seg = nr,
                          .seg_of_key = w.cseg, .roots = built, .leaf_cache = w.cache}));

    // ---- outputs ----
    rp_out_kernel<<<grid1d(dev, nr, 256), 256, 0, s>>>(bflags, nr, built, d_roots, more_flag, o_status, o_more);
    ctx->stats.launches++;
    CU(cudaMemcpyAsync(status, o_status, nr, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += nr;
    if (more) {
        CU(cudaMemcpyAsync(more, o_more, nr, cudaMemcpyDeviceToHost, s));
        ctx->stats.d2h_bytes += nr;
    }
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// Resident world state: account and storage proofs (phant_gpu_resident_state_prove, eth_getProof).  DESIGN.md §4.3f.
// The request's keys are staged in the diff layout and go through the apply's sort and classification; one proof key per
// requested key (each account key in the account trie, each slot key in its account's storage trie when the account is present
// with storage) goes through the witness's back end (rs_nodes), which leaves the node set sorted by digest; then one thread per
// proof walks its chain over that set (proof_chain.cuh): a counting pass, a scan, and a pass that writes the chains and the
// values read from the proven leaves.  Launches and read-backs follow trie depths, not how many keys are requested.
// ------------------------------------------------------------------------------------------------
namespace {

// the proof keys: candidate c < na is account c (sorted order) in trie 0, candidate na + j slot j (sorted order) in trie
// 1 + sacc[j]; a candidate is a proof key when its trie holds keys (w.ok)
__global__ void prf_key_flag_kernel(const uint32_t* __restrict__ sacc, uint32_t na, uint32_t ms, WitTries w, uint32_t* __restrict__ flag)
{
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c <= na + ms; c += gridDim.x * blockDim.x)
        flag[c] = c < na ? w.ok[0] : c < na + ms ? w.ok[1 + sacc[c - na]] : 0;
}
// the flagged candidates in order: already sorted by (trie, key)
__global__ void prf_key_list_kernel(const AccRow* __restrict__ arows, const SlotRow* __restrict__ srows, const uint32_t* __restrict__ sacc,
                                    uint32_t na, uint32_t ms, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos,
                                    uint8_t* __restrict__ pkeys, uint32_t* __restrict__ ptrie)
{
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < na + ms; c += gridDim.x * blockDim.x) {
        if (!flag[c]) continue;
        const uint4* k = reinterpret_cast<const uint4*>(c < na ? arows[c].key : srows[c - na].skey);
        uint4* d = reinterpret_cast<uint4*>(pkeys + 32ull * pos[c]);
        d[0] = k[0]; d[1] = k[1];
        ptrie[pos[c]] = c < na ? 0 : 1 + sacc[c - na];
    }
}

// proof p < na: account p of the request; proof na + j: slot j (the caller's order, as staged)
struct PrfIn {
    tn::PcSet set;
    const uint8_t *akeys, *skeys;
    const uint32_t* sacc;
    const uint32_t *rank, *alb; // sorted position of each requested account; its account row
    const uint8_t* ok;          // WitTries::ok: trie 1 + i holds keys (listed account i is present with storage)
    const AccRow* A;
    uint32_t na, ms;
    uint8_t root[32]; // the state root
};
__device__ __forceinline__ const uint8_t* prf_root(const PrfIn& in, uint32_t p)
{
    if (p < in.na) return in.root;
    const uint32_t i = in.rank[in.sacc[p - in.na]];
    return in.ok[1 + i] ? in.A[in.alb[i]].sroot : EMPTY_ROOT_D;
}
__device__ __forceinline__ const uint8_t* prf_key(const PrfIn& in, uint32_t p)
{
    return p < in.na ? in.akeys + 32ull * p : in.skeys + 32ull * (p - in.na);
}
// the held result, laid out in st->prf_res
struct PrfRes {
    uint64_t *node_index, *proof_first, *nonce;
    uint8_t *roots, *status, *bal, *sroot, *code, *svals;
    void take(Carve& c, uint64_t refs, uint32_t na, uint32_t ms)
    {
        const uint32_t np = na + ms;
        node_index = c.take<uint64_t>(refs); proof_first = c.take<uint64_t>(np + 1); roots = c.take<uint8_t>(32ull * np);
        status = c.take<uint8_t>(np); nonce = c.take<uint64_t>(na); bal = c.take<uint8_t>(32ull * na); sroot = c.take<uint8_t>(32ull * na);
        code = c.take<uint8_t>(32ull * na); svals = c.take<uint8_t>(32ull * ms);
    }
};
// chain lengths; bad[0]: a chain met a node that is missing or breaks the node rules
__global__ void prf_count_kernel(PrfIn in, uint64_t* __restrict__ len, uint32_t* __restrict__ bad)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < in.na + in.ms; p += gridDim.x * blockDim.x) {
        const tn::PcWalk w = tn::pc_walk(in.set, prf_root(in, p), EMPTY_ROOT_D, prf_key(in, p), nullptr);
        len[p] = w.len;
        if (w.status == tn::PC_BAD) bad[0] = 1;
    }
}
// the chains, roots, statuses and the values decoded from the proven leaves (P's decoders); bad[1]: a leaf value that does
// not decode
__global__ void prf_fill_kernel(PrfIn in, const uint64_t* __restrict__ first, PrfRes o, uint32_t* __restrict__ bad)
{
    const uint32_t np = in.na + in.ms;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p <= np; p += gridDim.x * blockDim.x) {
        o.proof_first[p] = first[p];
        if (p == np) continue;
        const uint8_t* root = prf_root(in, p);
        const tn::PcWalk w = tn::pc_walk(in.set, root, EMPTY_ROOT_D, prf_key(in, p), o.node_index + first[p]);
        for (int b = 0; b < 32; ++b) o.roots[32ull * p + b] = root[b];
        const uint8_t* v = in.set.bytes + w.val_off;
        bool ok = w.status == tn::PC_PRESENT;
        if (p < in.na) {
            AccountBody a{};
            if (ok && !decode_account_body(v, w.val_len, a)) { ok = false; bad[1] = 1; }
            o.nonce[p] = ok ? a.nonce : 0;
            for (uint32_t b = 0; b < 32; ++b) {
                o.bal[32ull * p + b] = ok && b >= 32 - a.bal_len ? v[a.bal_off + b - (32 - a.bal_len)] : 0;
                o.sroot[32ull * p + b] = ok ? v[a.root_off + b] : 0;
                o.code[32ull * p + b] = ok ? v[a.code_off + b] : 0;
            }
        } else {
            uint32_t off = 0, n = 0;
            if (ok && !tn::decode_slot_value(v, w.val_len, off, n)) { ok = false; bad[1] = 1; }
            const uint64_t j = p - in.na;
            for (uint32_t b = 0; b < 32; ++b) o.svals[32 * j + b] = ok && b >= 32 - n ? v[off + b - (32 - n)] : 0;
        }
        o.status[p] = w.status == tn::PC_PRESENT && !ok ? 0 : (uint8_t)w.status;
    }
}

// Host-side checks of a request (nothing is launched on a bad argument): host pointers only, sizes, slot owners.
int check_request_host(phant_gpu_ctx* ctx, const phant_gpu_proof_request* q)
{
    const uint64_t na64 = q->n_accounts, ms64 = q->n_slots;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID;
    if (na64 >= (1ull << 28) || ms64 >= (1ull << 28)) return PHANT_GPU_E_INVALID;
    if ((na64 && !q->account_keys32) || (ms64 && (!q->slot_account || !q->slot_keys32))) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({q->account_keys32, q->slot_account, q->slot_keys32})) return PHANT_GPU_E_INVALID;
    for (uint64_t j = 0; j < ms64; ++j)
        if (q->slot_account[j] >= na64) return PHANT_GPU_E_INVALID;
    return PHANT_GPU_OK;
}

// A checked request's keys copied to the device, into arrays the caller carved (akeys: n_accounts keys; sacc, skeys: n_slots).
int stage_request(phant_gpu_ctx* ctx, const phant_gpu_proof_request* q, uint8_t* akeys, uint32_t* sacc, uint8_t* skeys)
{
    cudaStream_t s = ctx->stream;
    const uint64_t na = q->n_accounts, ms = q->n_slots;
    CU(cudaMemcpyAsync(akeys, q->account_keys32, 32ull * na, cudaMemcpyHostToDevice, s));
    if (ms) {
        CU(cudaMemcpyAsync(sacc, q->slot_account, 4ull * ms, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(skeys, q->slot_keys32, 32ull * ms, cudaMemcpyHostToDevice, s));
    }
    ctx->stats.h2d_bytes += 32ull * na + 36ull * ms;
    return PHANT_GPU_OK;
}

// The proofs of a request (phant_gpu_resident_state_prove): the node set in st->wit_res, the rest in st->prf_res.
int rs_prove(phant_gpu_resident_state* st, const phant_gpu_proof_request* q)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    RC(check_request_host(ctx, q));
    const uint32_t na = (uint32_t)q->n_accounts, ms = (uint32_t)q->n_slots, npr = na + ms;
    st->prf_na = na;
    st->prf_ms = ms;
    if (na == 0) return PHANT_GPU_OK; // no proof (a slot needs an account)

    // ---- the keys staged in the diff layout: no flags (every account is read as it is), no values cross PCIe ----
    RsDiff dd;
    RC(carve(ctx, st->in, [&](Carve& c) { dd.take(c, na, ms); }));
    RC(stage_request(ctx, q, dd.akeys, dd.sacc, dd.skeys));
    CU(cudaMemsetAsync(dd.aflags, 0, na, s));
    if (ms) CU(cudaMemsetAsync(dd.svals, 0, 32ull * ms, s));

    // ---- the query front end; the proof keys: each requested key whose trie holds keys, already sorted by (trie, key) ----
    RsQuery rq;
    const RsSorted& f = rq.f;
    uint32_t *cflag, *cpos, *bad;
    uint64_t *plen, *pfirst;
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        rq.take(c, na, ms, st->nA);
        cflag = c.take<uint32_t>(npr + 1); cpos = c.take<uint32_t>(npr + 1);
        plen = c.take<uint64_t>(npr + 1); pfirst = c.take<uint64_t>(npr + 1); bad = c.take<uint32_t>(2);
    }));
    RC(rs_query_tries(st, dd, rq));
    prf_key_flag_kernel<<<grid1d(dev, npr + 1, 256), 256, 0, s>>>(f.sacc, na, ms, rq.w, cflag);
    RC(scan_u32(ctx, cflag, cpos, npr + 1));
    ctx->stats.launches++;
    uint32_t np = 0;
    RC(rs_query_check(st, rq, cpos + npr, &np));
    uint8_t* digests = nullptr;
    RC(rs_nodes(st, rq, np, [&](uint8_t* pkeys, uint32_t* ptrie) {
        prf_key_list_kernel<<<grid1d(dev, npr, 256), 256, 0, s>>>(f.arows, f.srows, f.sacc, na, ms, cflag, cpos, pkeys, ptrie);
        ctx->stats.launches++;
        return PHANT_GPU_OK;
    }, &digests));

    // ---- the chains: count, scan, fill ----
    PrfIn in;
    in.set = st->node_set(digests);
    in.akeys = dd.akeys; in.skeys = dd.skeys; in.sacc = dd.sacc;
    in.rank = f.rank; in.alb = f.alb; in.ok = rq.w.ok; in.A = st->acc_rows();
    in.na = na; in.ms = ms;
    memcpy(in.root, st->acct_sp.root, 32);
    CU(cudaMemsetAsync(bad, 0, 8, s));
    prf_count_kernel<<<grid1d(dev, npr, 128), 128, 0, s>>>(in, plen, bad);
    RC(scan_sizes(ctx, plen, pfirst, npr));
    uint64_t refs = 0;
    CU(cudaMemcpyAsync(&refs, pfirst + npr, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    PrfRes o;
    RC(carve(ctx, st->prf_res, [&](Carve& c) { o.take(c, refs, na, ms); }));
    prf_fill_kernel<<<grid1d(dev, npr + 1, 128), 128, 0, s>>>(in, pfirst, o, bad);
    uint32_t hb[2];
    CU(cudaMemcpyAsync(hb, bad, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    ctx->stats.d2h_bytes += 16;
    if (hb[0] || hb[1]) { // cannot happen: the node set holds every node on the proof keys' paths, encoded by the builders
        snprintf(ctx->last_error, sizeof ctx->last_error, "resident state: a proof chain met a missing or undecodable node");
        return PHANT_GPU_E_CUDA;
    }
    st->prf_refs = refs;
    return PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_resident_state_prove(phant_gpu_resident_state* st, const phant_gpu_proof_request* req, phant_gpu_proof_size* out)
{
    if (!req || !out) return PHANT_GPU_E_INVALID;
    RC(rs_build_result(st, RsResult::PROOFS, out, [&] { return rs_prove(st, req); }));
    out->n_nodes = st->wit_n;
    out->nodes_bytes = st->wit_bytes;
    out->n_refs = st->prf_refs;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_prove_copy(phant_gpu_resident_state* st, phant_gpu_proofs* out)
{
    if (!st || st->held != RsResult::PROOFS || !out) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    const uint64_t na = st->prf_na, ms = st->prf_ms, np = na + ms, refs = st->prf_refs;
    if (!out->node_off || !out->proof_first || (st->wit_bytes && !out->nodes) || (refs && !out->node_index)) return PHANT_GPU_E_INVALID;
    return rs_copy_result(st, {out->nodes, out->node_off, out->node_index, out->proof_first, out->roots32, out->status, out->nonce,
                               out->balance32, out->storage_root32, out->code_hash32, out->slot_vals32}, [&]() -> int {
        out->proof_first[0] = 0;
        RC(copy_node_set(st, out->node_off, out->nodes));
        if (!np) return PHANT_GPU_OK;
        Carve c{(uint8_t*)st->prf_res.ptr};
        PrfRes o;
        o.take(c, refs, (uint32_t)na, (uint32_t)ms);
        RC(copy_out(ctx, out->node_index, o.node_index, 8 * refs));
        RC(copy_out(ctx, out->proof_first, o.proof_first, 8 * (np + 1)));
        RC(copy_out(ctx, out->roots32, o.roots, 32 * np));
        RC(copy_out(ctx, out->status, o.status, np));
        RC(copy_out(ctx, out->nonce, o.nonce, 8 * na));
        RC(copy_out(ctx, out->balance32, o.bal, 32 * na));
        RC(copy_out(ctx, out->storage_root32, o.sroot, 32 * na));
        RC(copy_out(ctx, out->code_hash32, o.code, 32 * na));
        return copy_out(ctx, out->slot_vals32, o.svals, 32 * ms);
    });
}

// ------------------------------------------------------------------------------------------------
// Resident world state: trie nodes by path (phant_gpu_resident_state_trie_nodes, the snap protocol's GetTrieNodes).  DESIGN.md
// §4.3k.  prove's front end with paths in place of keys: the storage accounts are staged as the accounts of a request and go
// through the apply's sort and classification; each path becomes one proof key, its nibbles padded with zeros, in its trie;
// the keys are sorted by (trie, key) and rs_nodes rebuilds the node set on their paths (the node at a path lies on the path of
// every key that starts with it).  One thread per path then walks that set to the path's end (proof_chain.cuh, pc_node_at),
// and a count, a scan and a gather put the served nodes into request-order CSR.  Launches and read-backs follow trie depths,
// not how many paths are requested.
// ------------------------------------------------------------------------------------------------
namespace {

// proof-key candidate p: path p's first plen[p] nibbles padded with zeros, in trie 0 or 1 + its storage account's rank, or
// NONE when that trie holds no key; count[0]: the candidates that are proof keys
__global__ void tnd_keys_kernel(const uint8_t* __restrict__ paths, const uint8_t* __restrict__ plen, const uint32_t* __restrict__ ptrie,
                                uint32_t n, const uint32_t* __restrict__ rank, WitTries w, uint8_t* __restrict__ ckeys,
                                uint32_t* __restrict__ cseg, uint32_t* __restrict__ count)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const uint32_t t = ptrie[p] ? 1 + rank[ptrie[p] - 1] : 0, L = plen[p];
        for (uint32_t b = 0; b < 32; ++b) {
            const uint8_t keep = 2 * b + 2 <= L ? 0xff : 2 * b + 1 == L ? 0xf0 : 0;
            ckeys[32ull * p + b] = paths[32ull * p + b] & keep;
        }
        cseg[p] = w.ok[t] ? t : NONE;
        if (w.ok[t]) atomicAdd(count, 1u);
    }
}

struct TndIn {
    tn::PcSet set;
    const uint8_t *paths, *plen;
    const uint32_t* ptrie;
    const uint32_t *rank, *alb; // sorted position of each storage account; its account row
    const uint8_t* ok;          // WitTries::ok
    const AccRow* A;
    uint32_t n;
    uint8_t root[32]; // the state root
};
// per path: status, the served node's index in the set and its length; count[1]: a walk met a node that is missing or breaks
// the node rules; count[2]: the paths served
__global__ void tnd_walk_kernel(TndIn in, uint8_t* __restrict__ status, uint32_t* __restrict__ index, uint64_t* __restrict__ size,
                                uint32_t* __restrict__ count)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < in.n; p += gridDim.x * blockDim.x) {
        const uint32_t j = in.ptrie[p], i = j ? in.rank[j - 1] : 0;
        const uint8_t* root = j == 0 ? in.root : in.ok[1 + i] ? in.A[in.alb[i]].sroot : EMPTY_ROOT_D;
        const tn::PcAt a = tn::pc_node_at(in.set, root, EMPTY_ROOT_D, in.paths + 32ull * p, in.plen[p]);
        const bool hit = a.status == tn::PC_PRESENT;
        if (a.status == tn::PC_BAD) count[1] = 1;
        if (hit) atomicAdd(count + 2, 1u);
        status[p] = hit ? 1 : 2;
        index[p] = a.index;
        size[p] = hit ? in.set.off[a.index + 1] - in.set.off[a.index] : 0;
    }
}

// the held result, laid out in st->tnd_res
struct TndRes {
    uint8_t* status;
    uint64_t* node_off;
    uint8_t* bytes;
    void take(Carve& c, uint32_t n, uint64_t nb)
    {
        status = c.take<uint8_t>(n); node_off = c.take<uint64_t>(n + 1); bytes = c.take<uint8_t>(nb);
    }
};
// one warp per path: its status, offset and node bytes into the result
__global__ void tnd_gather_kernel(tn::PcSet set, const uint8_t* __restrict__ status, const uint32_t* __restrict__ index,
                                  const uint64_t* __restrict__ offs, uint32_t n, TndRes o)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p <= n; p += (gridDim.x * blockDim.x) >> 5) {
        if (lane == 0) {
            o.node_off[p] = offs[p];
            if (p < n) o.status[p] = status[p];
        }
        if (p == n || status[p] != 1) continue;
        const uint8_t* src = set.bytes + set.off[index[p]];
        const uint64_t len = offs[p + 1] - offs[p];
        for (uint64_t b = lane; b < len; b += 32) o.bytes[offs[p] + b] = src[b];
    }
}

// Host-side checks of a request (nothing is launched on a bad argument): host pointers only, sizes, path lengths, owners.
int check_trie_node_request(phant_gpu_ctx* ctx, const phant_gpu_trie_node_request* q)
{
    const uint64_t n = q->n_paths, m = q->n_storage_accounts;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID;
    if (n > (1ull << 28) || m > (1ull << 28)) return PHANT_GPU_E_INVALID;
    if (n && (!q->paths32 || !q->path_len)) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({q->paths32, q->path_len, q->path_trie, q->storage_account32})) return PHANT_GPU_E_INVALID;
    bool storage = false;
    for (uint64_t p = 0; p < n; ++p) {
        if (q->path_len[p] > 64) return PHANT_GPU_E_INVALID;
        if (!q->path_trie) continue;
        if (q->path_trie[p] > m) return PHANT_GPU_E_INVALID;
        storage |= q->path_trie[p] > 0;
    }
    return storage && !q->storage_account32 ? PHANT_GPU_E_INVALID : PHANT_GPU_OK;
}

// The trie nodes of a request (phant_gpu_resident_state_trie_nodes): the node set in st->wit_res (scratch here), the result in
// st->tnd_res.
int rs_trie_nodes(phant_gpu_resident_state* st, const phant_gpu_trie_node_request* q)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    RC(check_trie_node_request(ctx, q));
    // no storage account is read when none is named (storage_account32 may then be NULL)
    const uint32_t n = (uint32_t)q->n_paths, na = q->storage_account32 ? (uint32_t)q->n_storage_accounts : 0;
    st->tnd_n = n;
    if (n == 0) return PHANT_GPU_OK;

    // ---- the request on the device: the storage accounts in the diff layout with no flags and no slots, then the paths ----
    RsDiff dd;
    uint8_t *paths, *plen;
    uint32_t* ptrie;
    RC(carve(ctx, st->in, [&](Carve& c) {
        dd.take(c, na, 0);
        paths = c.take<uint8_t>(32ull * n); plen = c.take<uint8_t>(n); ptrie = c.take<uint32_t>(n);
    }));
    if (na) {
        CU(cudaMemcpyAsync(dd.akeys, q->storage_account32, 32ull * na, cudaMemcpyHostToDevice, s));
        CU(cudaMemsetAsync(dd.aflags, 0, na, s));
    }
    CU(cudaMemcpyAsync(paths, q->paths32, 32ull * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(plen, q->path_len, n, cudaMemcpyHostToDevice, s));
    if (q->path_trie) CU(cudaMemcpyAsync(ptrie, q->path_trie, 4ull * n, cudaMemcpyHostToDevice, s));
    else CU(cudaMemsetAsync(ptrie, 0, 4ull * n, s));
    ctx->stats.h2d_bytes += 32ull * na + 33ull * n + (q->path_trie ? 4ull * n : 0);

    // ---- the query front end over the accounts (no slot: counters[1] stays 0); one proof-key candidate per path ----
    RsQuery rq;
    const RsSorted& f = rq.f;
    uint8_t *ckeys, *status;
    uint32_t *cseg, *cperm, *index, *count;
    uint64_t *size, *offs;
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        rq.take(c, na, 0, st->nA);
        ckeys = c.take<uint8_t>(32ull * n); cseg = c.take<uint32_t>(n); cperm = c.take<uint32_t>(n);
        status = c.take<uint8_t>(n); index = c.take<uint32_t>(n); size = c.take<uint64_t>(n + 1); offs = c.take<uint64_t>(n + 1);
        count = c.take<uint32_t>(4);
    }));
    RC(rs_query_tries(st, dd, rq));
    CU(cudaMemsetAsync(count, 0, 16, s));
    tnd_keys_kernel<<<grid1d(dev, n, 128), 128, 0, s>>>(paths, plen, ptrie, n, f.rank, rq.w, ckeys, cseg, count);
    ctx->stats.launches++;
    uint32_t np = 0;
    RC(rs_query_check(st, rq, count, &np)); // a storage account twice
    uint8_t* digests = nullptr;
    RC(rs_nodes(st, rq, np, [&](uint8_t* pkeys, uint32_t* pktrie) { return rs_candidate_keys(st, ckeys, cseg, cperm, n, np, pkeys, pktrie); },
                &digests));

    // ---- the walks, then the served nodes in request order: count, scan, gather ----
    TndIn in;
    in.set = st->node_set(digests);
    in.paths = paths; in.plen = plen; in.ptrie = ptrie;
    in.rank = f.rank; in.alb = f.alb; in.ok = rq.w.ok; in.A = st->acc_rows();
    in.n = n;
    memcpy(in.root, st->acct_sp.root, 32);
    tnd_walk_kernel<<<grid1d(dev, n, 128), 128, 0, s>>>(in, status, index, size, count);
    RC(scan_sizes(ctx, size, offs, n));
    uint64_t nb = 0;
    uint32_t hc[4];
    CU(cudaMemcpyAsync(&nb, offs + n, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(hc, count, 16, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches++;
    ctx->stats.d2h_bytes += 24;
    if (hc[1]) { // cannot happen: the node set holds every node on the padded paths, encoded by the builders
        snprintf(ctx->last_error, sizeof ctx->last_error, "resident state: a trie-node walk met a missing or undecodable node");
        return PHANT_GPU_E_CUDA;
    }
    TndRes o;
    RC(carve(ctx, st->tnd_res, [&](Carve& c) { o.take(c, n, nb); }));
    tnd_gather_kernel<<<grid1d(dev, n + 1, 256, 32), 256, 0, s>>>(in.set, status, index, offs, n, o);
    ctx->stats.launches++;
    st->tnd_nodes = hc[2];
    st->tnd_bytes = nb;
    return PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_resident_state_trie_nodes(phant_gpu_resident_state* st, const phant_gpu_trie_node_request* req,
                                                   phant_gpu_witness_size* out)
{
    if (!req || !out) return PHANT_GPU_E_INVALID;
    RC(rs_build_result(st, RsResult::TRIE_NODES, out, [&] { return rs_trie_nodes(st, req); }));
    out->n_nodes = st->tnd_nodes;
    out->nodes_bytes = st->tnd_bytes;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_trie_nodes_copy(phant_gpu_resident_state* st, phant_gpu_trie_nodes* out)
{
    if (!st || st->held != RsResult::TRIE_NODES || !out) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    const uint32_t n = st->tnd_n;
    if (!out->node_off || (n && !out->status) || (st->tnd_bytes && !out->nodes)) return PHANT_GPU_E_INVALID;
    return rs_copy_result(st, {out->status, out->node_off, out->nodes}, [&]() -> int {
        out->node_off[0] = 0;
        if (!n) return PHANT_GPU_OK;
        Carve c{(uint8_t*)st->tnd_res.ptr};
        TndRes o;
        o.take(c, n, st->tnd_bytes);
        RC(copy_out(ctx, out->status, o.status, n));
        RC(copy_out(ctx, out->node_off, o.node_off, 8ull * (n + 1)));
        return copy_out(ctx, out->nodes, o.bytes, st->tnd_bytes);
    });
}

// ------------------------------------------------------------------------------------------------
// Resident world state: snap range answers (phant_gpu_resident_state_snap_ranges, the snap protocol's GetAccountRange and
// GetStorageRanges).  DESIGN.md §4.3m.  range's back-0 path with geth's byte cuts (snap_range.cuh): one thread per request
// finds its candidate run in the account row table or, account after account, in the slot table, bounded by what its budget
// can return; one thread per candidate sizes its entry; a scan of the sizes gives every request's cut by binary search.  The
// proof keys (each account request's origin and last key, each proved storage account's origin and last key) go through
// prove's front end and rs_nodes; one thread per request walks its two chains over that set and merges them into the wire
// list.  Then one fill writes keys, slim or slot bodies and the lists.  Launches do not grow with the number of requests.
// ------------------------------------------------------------------------------------------------
namespace {

// the requests of one call: r < n is account request r, r >= n storage request r - n over accounts [first[q], first[q + 1])
struct SnpReq {
    const uint8_t *origin, *limit; // (n + m) x 32
    const uint64_t* bytes;         // n + m
    const uint64_t* first;         // m + 1
    const uint8_t* accts;          // M x 32
    const uint32_t* uidx;          // M: the account's place among the distinct accounts staged for the query front end
    uint32_t n, m;
    uint64_t M;
};
// candidate segments: r < n is account request r, n + k storage account k; lo: first row, cnt: candidates, coff: their
// offsets, run (M): the account's whole run
struct SnpCand {
    uint32_t* lo;
    uint64_t *cnt, *coff, *run;
};
// the held result, laid out in st->snp_res
struct SnpRes {
    uint64_t *afirst, *aoff, *sfirst, *slot_first, *soff, *pfirst, *node_index;
    uint8_t *akeys, *abodies, *skeys, *sbodies;
    void take(Carve& c, uint32_t n, uint32_t m, uint64_t ea, uint64_t ab, uint64_t ns, uint64_t es, uint64_t sb, uint64_t refs)
    {
        afirst = c.take<uint64_t>(n + 1); akeys = c.take<uint8_t>(32 * ea); aoff = c.take<uint64_t>(ea + 1); abodies = c.take<uint8_t>(ab);
        sfirst = c.take<uint64_t>(m + 1); slot_first = c.take<uint64_t>(ns + 1); skeys = c.take<uint8_t>(32 * es);
        soff = c.take<uint64_t>(es + 1); sbodies = c.take<uint8_t>(sb); pfirst = c.take<uint64_t>(n + m + 1);
        node_index = c.take<uint64_t>(refs);
    }
};

// every request's candidates
__global__ void snp_window_kernel(SnpReq q, const KRow* __restrict__ krows, uint32_t nK, const SlotRow* __restrict__ S, uint32_t nS, SnpCand c)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < q.n + q.m; r += gridDim.x * blockDim.x) {
        if (r < q.n) {
            tn::snp_account_window(krows, nK, q.origin + 32ull * r, q.limit + 32ull * r, q.bytes[r], c.lo[r], c.cnt[r]);
            continue;
        }
        const uint64_t F = q.first[r - q.n], G = q.first[r - q.n + 1];
        tn::snp_storage_window(S, nS, q.accts + 32 * F, G - F, q.origin + 32ull * r, q.limit + 32ull * r, q.bytes[r], c.lo + q.n + F, c.run + F,
                               c.cnt + q.n + F);
    }
}

// candidate j's entry size; bad: an account leaf that does not decode
__global__ void snp_size_kernel(SnpReq q, const KRow* __restrict__ krows, const uint8_t* __restrict__ arena, const SlotRow* __restrict__ S,
                                SnpCand c, uint64_t C, uint64_t* __restrict__ size, uint32_t* __restrict__ bad)
{
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < C; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = tn::rg_segment(c.coff, q.n + q.M, j), row = c.lo[r] + (j - c.coff[r]);
        uint32_t len;
        if (r < q.n) {
            len = tn::snp_slim(arena + krows[row].off, krows[row].len, nullptr);
            if (!len) *bad = 1;
        } else {
            len = tn::snp_slot_body(S[row].val, nullptr);
        }
        size[j] = 32 + len;
    }
}

// Every request's cut (x: the scan of the candidates' sizes): entries and body bytes per segment, storage accounts served per
// storage request, and its proof-key candidates 2r, 2r + 1 (origin, last key) in trie 0 or in 1 + the proved account's
// sorted rank, NONE when there is none or that trie holds no key; count[0]: the proof keys
__global__ void snp_cut_kernel(SnpReq q, const KRow* __restrict__ krows, const SlotRow* __restrict__ S, SnpCand c, const uint64_t* __restrict__ x,
                               WitTries w, const uint32_t* __restrict__ rank, uint64_t* __restrict__ ent, uint64_t* __restrict__ body,
                               uint64_t* __restrict__ served, uint8_t* __restrict__ ckeys, uint32_t* __restrict__ cseg, uint32_t* __restrict__ count)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < q.n + q.m; r += gridDim.x * blockDim.x) {
        const uint32_t c0 = 2 * r;
        cseg[c0] = cseg[c0 + 1] = NONE;
        const uint8_t* origin = q.origin + 32ull * r;
        uint32_t got = 0;
        if (r < q.n) {
            const uint64_t e = tn::snp_account_cut(x + c.coff[r], c.cnt[r], q.bytes[r]);
            ent[r] = e;
            body[r] = x[c.coff[r] + e] - x[c.coff[r]] - 32 * e;
            if (w.ok[0]) {
                wit_put(ckeys, cseg, c0, origin, 0);
                ++got;
                if (e) { wit_put(ckeys, cseg, c0 + 1, krows[c.lo[r] + e - 1].key, 0); ++got; }
            }
        } else {
            const uint64_t F = q.first[r - q.n], G = q.first[r - q.n + 1], R = q.n + F;
            bool set = false;
            for (int b = 0; b < 32; ++b) set |= origin[b] != 0;
            const tn::SnpServe sv = tn::snp_storage_cut(x + c.coff[R], c.cnt + R, c.run + F, G - F, set, q.bytes[r], ent + R);
            for (uint64_t k = R; k < q.n + G; ++k) body[k] = x[c.coff[k] + ent[k]] - x[c.coff[k]] - 32 * ent[k];
            served[r - q.n] = sv.served;
            if (sv.proved != tn::SNP_NONE) {
                const uint64_t k = F + sv.proved;
                const uint32_t t = 1 + rank[q.uidx[k]];
                if (w.ok[t]) {
                    wit_put(ckeys, cseg, c0, origin, t); // a later account's origin is 0
                    if (sv.proved)
                        for (int b = 0; b < 32; ++b) ckeys[32ull * c0 + b] = 0;
                    ++got;
                    if (ent[q.n + k]) { wit_put(ckeys, cseg, c0 + 1, S[c.lo[q.n + k] + ent[q.n + k] - 1].skey, t); ++got; }
                }
            }
        }
        if (got) atomicAdd(count, got);
    }
}

// the proof chains: candidate c (cseg: its trie, NONE for no chain) walked over the node set from its trie's root
struct SnpChains {
    tn::PcSet set;
    const uint8_t* ckeys;
    const uint32_t* cseg;
    const uint32_t* alb; // the staged accounts' rows, by sorted rank
    const AccRow* A;
    uint32_t nc;
    uint8_t root[32]; // the state root
};
__device__ __forceinline__ uint32_t snp_chain(const SnpChains& in, uint32_t c, uint64_t* chain, uint32_t* bad)
{
    const uint32_t t = in.cseg[c];
    if (t == NONE) return 0;
    const tn::PcWalk wk = tn::pc_walk(in.set, t ? in.A[in.alb[t - 1]].sroot : in.root, EMPTY_ROOT_D, in.ckeys + 32ull * c, chain);
    if (wk.status == tn::PC_BAD) *bad = 1;
    return wk.len;
}
__global__ void snp_chain_len_kernel(SnpChains in, uint64_t* __restrict__ len, uint32_t* __restrict__ bad)
{
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < in.nc; c += gridDim.x * blockDim.x) len[c] = snp_chain(in, c, nullptr, bad);
}
// entry i of request r's second chain is listed when neither its first chain nor an earlier entry of the second holds it
__device__ __forceinline__ bool snp_new_in_last(const uint64_t* a, uint64_t na, const uint64_t* b, uint64_t i)
{
    for (uint64_t k = 0; k < na; ++k)
        if (a[k] == b[i]) return false;
    for (uint64_t k = 0; k < i; ++k)
        if (b[k] == b[i]) return false;
    return true;
}
// per request: its two chains into tmp (offsets toff), and the length of its merged list
__global__ void snp_chain_kernel(SnpChains in, const uint64_t* __restrict__ toff, uint64_t* __restrict__ tmp, uint64_t* __restrict__ mlen,
                                 uint32_t* __restrict__ bad)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < in.nc / 2; r += gridDim.x * blockDim.x) {
        uint64_t *a = tmp + toff[2 * r], *b = tmp + toff[2 * r + 1];
        const uint64_t na = snp_chain(in, 2 * r, a, bad), nb = snp_chain(in, 2 * r + 1, b, bad);
        uint64_t len = na;
        for (uint64_t i = 0; i < nb; ++i) len += snp_new_in_last(a, na, b, i);
        mlen[r] = len;
    }
}
// per request: its merged list into node_index, and proof_first
__global__ void snp_proof_fill_kernel(const uint64_t* __restrict__ toff, const uint64_t* __restrict__ tmp, const uint64_t* __restrict__ mfirst,
                                      uint32_t R, SnpRes o)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= R; r += gridDim.x * blockDim.x) {
        o.pfirst[r] = mfirst[r];
        if (r == R) continue;
        const uint64_t *a = tmp + toff[2 * r], *b = tmp + toff[2 * r + 1];
        const uint64_t na = toff[2 * r + 1] - toff[2 * r], nb = toff[2 * r + 2] - toff[2 * r + 1];
        uint64_t* out = o.node_index + mfirst[r];
        for (uint64_t i = 0; i < na; ++i) *out++ = a[i];
        for (uint64_t i = 0; i < nb; ++i)
            if (snp_new_in_last(a, na, b, i)) *out++ = b[i];
    }
}

// entry e (E: entry offsets, B: body offsets over the n + M segments): its key and body
__global__ void snp_fill_kernel(SnpReq q, const KRow* __restrict__ krows, const uint8_t* __restrict__ arena, const SlotRow* __restrict__ S,
                                SnpCand c, const uint64_t* __restrict__ x, const uint64_t* __restrict__ E, const uint64_t* __restrict__ B, SnpRes o)
{
    const uint64_t nseg = q.n + q.M, ea = E[q.n], total = E[nseg];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        o.aoff[ea] = B[q.n];
        o.soff[total - ea] = B[nseg] - B[q.n];
    }
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = tn::rg_segment(E, nseg, e), t = e - E[r], row = c.lo[r] + t;
        const uint64_t boff = B[r] + (x[c.coff[r] + t] - x[c.coff[r]]) - 32 * t;
        const uint4* k = reinterpret_cast<const uint4*>(r < q.n ? krows[row].key : S[row].skey);
        uint4* d = reinterpret_cast<uint4*>(r < q.n ? o.akeys + 32 * e : o.skeys + 32 * (e - ea));
        d[0] = k[0]; d[1] = k[1];
        if (r < q.n) {
            o.aoff[e] = boff;
            tn::snp_slim(arena + krows[row].off, krows[row].len, o.abodies + boff);
        } else {
            o.soff[e - ea] = boff - B[q.n];
            tn::snp_slot_body(S[row].val, o.sbodies + boff - B[q.n]);
        }
    }
}
// the answers' offsets: account_first, served_first, and slot_first over the ns served accounts
__global__ void snp_index_kernel(SnpReq q, const uint64_t* __restrict__ E, const uint64_t* __restrict__ SF, uint64_t ns, SnpRes o)
{
    const uint64_t top = ns > q.n ? (ns > q.m ? ns : q.m) : (q.n > q.m ? q.n : q.m);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= top; i += (uint64_t)gridDim.x * blockDim.x) {
        if (i <= q.n) o.afirst[i] = E[i];
        if (i <= q.m) o.sfirst[i] = SF[i];
        if (i < ns) {
            const uint64_t r = tn::rg_segment(SF, q.m, i), k = q.first[r] + i - SF[r];
            o.slot_first[i] = E[q.n + k] - E[q.n];
        } else if (i == ns) {
            o.slot_first[i] = E[q.n + q.M] - E[q.n];
        }
    }
}

// Host-side checks of a request (nothing is launched on a bad argument): host pointers only, sizes, storage_first.
int check_snap_request(phant_gpu_ctx* ctx, const phant_gpu_snap_request* q)
{
    const uint64_t n = q->n_account_requests, m = q->n_storage_requests;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID;
    if (n > (1ull << 28) || m > (1ull << 28)) return PHANT_GPU_E_INVALID;
    if (n && (!q->account_origin32 || !q->account_limit32 || !q->account_bytes)) return PHANT_GPU_E_INVALID;
    if (m && (!q->storage_first || !q->storage_origin32 || !q->storage_limit32 || !q->storage_bytes)) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({q->account_origin32, q->account_limit32, q->account_bytes, q->storage_first, q->storage_accounts32, q->storage_origin32,
                    q->storage_limit32, q->storage_bytes}))
        return PHANT_GPU_E_INVALID;
    if (!m) return PHANT_GPU_OK;
    if (q->storage_first[0] != 0) return PHANT_GPU_E_INVALID;
    for (uint64_t i = 0; i < m; ++i)
        if (q->storage_first[i + 1] < q->storage_first[i]) return PHANT_GPU_E_INVALID;
    const uint64_t M = q->storage_first[m];
    if (M > (1ull << 28) || (M && !q->storage_accounts32)) return PHANT_GPU_E_INVALID;
    return host_ptrs({q->storage_accounts32}) ? PHANT_GPU_OK : PHANT_GPU_E_INVALID;
}

// The answers of a request (phant_gpu_resident_state_snap_ranges): the node set in st->wit_res, the rest in st->snp_res.
int rs_snap_ranges(phant_gpu_resident_state* st, const phant_gpu_snap_request* hq)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    RC(check_snap_request(ctx, hq));
    const uint32_t n = (uint32_t)hq->n_account_requests, m = (uint32_t)hq->n_storage_requests, R = n + m;
    const uint64_t M = m ? hq->storage_first[m] : 0, nseg = n + M;
    st->snp_n = n;
    st->snp_m = m;
    if (R == 0) return PHANT_GPU_OK;

    // ---- the distinct storage accounts, sorted on the host: a proved account's trie needs its account in the query, and the
    // query front end takes each account once ----
    std::vector<uint32_t> order(M), uidx(M);
    for (uint64_t k = 0; k < M; ++k) order[k] = (uint32_t)k;
    const uint8_t* ha = hq->storage_accounts32;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return memcmp(ha + 32ull * a, ha + 32ull * b, 32) < 0; });
    std::vector<uint8_t> ukeys;
    for (uint64_t i = 0; i < M; ++i) {
        const uint32_t k = order[i];
        if (!i || memcmp(ha + 32ull * order[i - 1], ha + 32ull * k, 32) != 0) ukeys.insert(ukeys.end(), ha + 32ull * k, ha + 32ull * k + 32);
        uidx[k] = (uint32_t)(ukeys.size() / 32 - 1);
    }
    const uint32_t U = (uint32_t)(ukeys.size() / 32);

    // ---- the request on the device: the distinct accounts in the diff layout (no flags, no slots), then the requests ----
    RsDiff dd;
    SnpReq q{};
    SnpCand c;
    uint8_t *origin, *limit, *accts, *ckeys;
    uint64_t *bytes, *first, *ent, *E, *body, *B, *served, *SF, *clen, *toff, *mlen, *mfirst;
    uint32_t *duidx, *cseg, *cperm, *count;
    RC(carve(ctx, st->in, [&](Carve& cv) {
        dd.take(cv, U, 0);
        origin = cv.take<uint8_t>(32ull * R); limit = cv.take<uint8_t>(32ull * R); bytes = cv.take<uint64_t>(R); first = cv.take<uint64_t>(m + 1);
        accts = cv.take<uint8_t>(32 * M); duidx = cv.take<uint32_t>(M);
        c.lo = cv.take<uint32_t>(nseg); c.cnt = cv.take<uint64_t>(nseg + 1); c.coff = cv.take<uint64_t>(nseg + 1); c.run = cv.take<uint64_t>(M);
        ent = cv.take<uint64_t>(nseg + 1); E = cv.take<uint64_t>(nseg + 1); body = cv.take<uint64_t>(nseg + 1); B = cv.take<uint64_t>(nseg + 1);
        served = cv.take<uint64_t>(m + 1); SF = cv.take<uint64_t>(m + 1);
        ckeys = cv.take<uint8_t>(64ull * R); cseg = cv.take<uint32_t>(2ull * R); cperm = cv.take<uint32_t>(2ull * R);
        clen = cv.take<uint64_t>(2ull * R + 1); toff = cv.take<uint64_t>(2ull * R + 1); mlen = cv.take<uint64_t>(R + 1); mfirst = cv.take<uint64_t>(R + 1);
        count = cv.take<uint32_t>(4);
    }));
    if (U) {
        CU(cudaMemcpyAsync(dd.akeys, ukeys.data(), 32ull * U, cudaMemcpyHostToDevice, s));
        CU(cudaMemsetAsync(dd.aflags, 0, U, s));
    }
    if (n) {
        CU(cudaMemcpyAsync(origin, hq->account_origin32, 32ull * n, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(limit, hq->account_limit32, 32ull * n, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(bytes, hq->account_bytes, 8ull * n, cudaMemcpyHostToDevice, s));
    }
    if (m) {
        CU(cudaMemcpyAsync(origin + 32ull * n, hq->storage_origin32, 32ull * m, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(limit + 32ull * n, hq->storage_limit32, 32ull * m, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(bytes + n, hq->storage_bytes, 8ull * m, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(first, hq->storage_first, 8ull * (m + 1), cudaMemcpyHostToDevice, s));
    }
    if (M) {
        CU(cudaMemcpyAsync(accts, ha, 32 * M, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(duidx, uidx.data(), 4 * M, cudaMemcpyHostToDevice, s));
    }
    ctx->stats.h2d_bytes += 32ull * U + 72ull * R + (m ? 8ull * (m + 1) : 0) + 36 * M;
    q.origin = origin; q.limit = limit; q.bytes = bytes; q.first = first; q.accts = accts; q.uidx = duidx;
    q.n = n; q.m = m; q.M = M;

    // ---- the candidates of every request, and how many there are ----
    const KRow* krows = st->acct_rows();
    const uint32_t nK = (uint32_t)st->acct_sp.n;
    const SlotRow* S = st->slot_table();
    snp_window_kernel<<<grid1d(dev, R, 128), 128, 0, s>>>(q, krows, nK, S, st->nS, c);
    RC(scan_sizes(ctx, c.cnt, c.coff, nseg));
    uint64_t C = 0;
    RC(copy_out(ctx, &C, c.coff + nseg, 8));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;

    // ---- the query front end over the distinct accounts; sizes, their scan and every request's cut ----
    RsQuery rq;
    uint64_t *size, *x;
    RC(carve(ctx, st->dirty, [&](Carve& cv) {
        rq.take(cv, U, 0, st->nA);
        size = cv.take<uint64_t>(C + 1); x = cv.take<uint64_t>(C + 1);
    }));
    RC(rs_query_tries(st, dd, rq));
    CU(cudaMemsetAsync(count, 0, 16, s));
    if (C) {
        snp_size_kernel<<<grid1d(dev, C, 256), 256, 0, s>>>(q, krows, st->acct_arena(), S, c, C, size, count + 1);
        ctx->stats.launches++;
    }
    RC(scan_sizes(ctx, size, x, C));
    snp_cut_kernel<<<grid1d(dev, R, 128), 128, 0, s>>>(q, krows, S, c, x, rq.w, rq.f.rank, ent, body, served, ckeys, cseg, count);
    RC(scan_sizes(ctx, ent, E, nseg));
    RC(scan_sizes(ctx, body, B, nseg));
    RC(scan_sizes(ctx, served, SF, m));
    ctx->stats.launches += 5;
    uint64_t hE[2], hB[2], ns = 0;
    uint32_t hc[4];
    RC(copy_out(ctx, hE, E + n, 8));
    RC(copy_out(ctx, hE + 1, E + nseg, 8));
    RC(copy_out(ctx, hB, B + n, 8));
    RC(copy_out(ctx, hB + 1, B + nseg, 8));
    RC(copy_out(ctx, &ns, SF + m, 8));
    RC(copy_out(ctx, hc, count, 16));
    CU(cudaStreamSynchronize(s));
    if (hc[1]) return rs_undecodable_leaf(ctx);
    const uint32_t np = hc[0];

    // ---- the node set on the proof keys, then each request's two chains merged ----
    uint8_t* digests = nullptr;
    RC(rs_nodes(st, rq, np, [&](uint8_t* pkeys, uint32_t* ptrie) { return rs_candidate_keys(st, ckeys, cseg, cperm, 2 * R, np, pkeys, ptrie); },
                &digests));
    SnpChains in;
    in.set = st->node_set(digests);
    in.ckeys = ckeys; in.cseg = cseg; in.alb = rq.f.alb; in.A = st->acc_rows();
    in.nc = 2 * R;
    memcpy(in.root, st->acct_sp.root, 32);
    CU(cudaMemsetAsync(count + 2, 0, 4, s));
    snp_chain_len_kernel<<<grid1d(dev, 2 * R, 128), 128, 0, s>>>(in, clen, count + 2);
    RC(scan_sizes(ctx, clen, toff, 2ull * R));
    uint64_t T = 0;
    RC(copy_out(ctx, &T, toff + 2ull * R, 8));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    uint64_t* tmp;
    RC(carve(ctx, st->forest, [&](Carve& cv) { tmp = cv.take<uint64_t>(T); }));
    snp_chain_kernel<<<grid1d(dev, R, 128), 128, 0, s>>>(in, toff, tmp, mlen, count + 2);
    RC(scan_sizes(ctx, mlen, mfirst, R));
    uint64_t refs = 0;
    uint32_t hbad = 0;
    RC(copy_out(ctx, &refs, mfirst + R, 8));
    RC(copy_out(ctx, &hbad, count + 2, 4));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    if (hbad) { // cannot happen: the node set holds every node on the proof keys' paths, encoded by the builders
        snprintf(ctx->last_error, sizeof ctx->last_error, "resident state: a snap proof chain met a missing or undecodable node");
        return PHANT_GPU_E_CUDA;
    }

    // ---- the answers ----
    const uint64_t ea = hE[0], es = hE[1] - hE[0], ab = hB[0], sb = hB[1] - hB[0];
    SnpRes o;
    RC(carve(ctx, st->snp_res, [&](Carve& cv) { o.take(cv, n, m, ea, ab, ns, es, sb, refs); }));
    if (ea + es) {
        snp_fill_kernel<<<grid1d(dev, ea + es, 128), 128, 0, s>>>(q, krows, st->acct_arena(), S, c, x, E, B, o);
        ctx->stats.launches++;
    } else {
        CU(cudaMemsetAsync(o.aoff, 0, 8, s));
        CU(cudaMemsetAsync(o.soff, 0, 8, s));
    }
    const uint64_t top = ns > n ? (ns > m ? ns : m) : (n > m ? n : m);
    snp_index_kernel<<<grid1d(dev, top + 1, 256), 256, 0, s>>>(q, E, SF, ns, o);
    snp_proof_fill_kernel<<<grid1d(dev, R + 1, 128), 128, 0, s>>>(toff, tmp, mfirst, R, o);
    ctx->stats.launches += 2;
    st->snp_ea = ea; st->snp_ab = ab; st->snp_ns = ns; st->snp_es = es; st->snp_sb = sb; st->snp_refs = refs;
    return PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_resident_state_snap_ranges(phant_gpu_resident_state* st, const phant_gpu_snap_request* req, phant_gpu_snap_size* out)
{
    if (!req || !out) return PHANT_GPU_E_INVALID;
    RC(rs_build_result(st, RsResult::SNAP_RANGES, out, [&] { return rs_snap_ranges(st, req); }));
    out->n_accounts = st->snp_ea;
    out->account_bytes = st->snp_ab;
    out->n_served = st->snp_ns;
    out->n_slots = st->snp_es;
    out->slot_bytes = st->snp_sb;
    out->n_nodes = st->wit_n;
    out->nodes_bytes = st->wit_bytes;
    out->n_refs = st->snp_refs;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_snap_ranges_copy(phant_gpu_resident_state* st, phant_gpu_snap_ranges* out)
{
    if (!st || st->held != RsResult::SNAP_RANGES || !out) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    const uint32_t n = st->snp_n, m = st->snp_m;
    const uint64_t ea = st->snp_ea, es = st->snp_es, ns = st->snp_ns;
    if (!out->account_first || !out->account_body_off || !out->served_first || !out->slot_first || !out->slot_body_off || !out->proof_first ||
        !out->node_off || (ea && !out->account_keys32) || (st->snp_ab && !out->account_bodies) || (es && !out->slot_keys32) ||
        (st->snp_sb && !out->slot_bodies) || (st->snp_refs && !out->node_index) || (st->wit_bytes && !out->nodes))
        return PHANT_GPU_E_INVALID;
    return rs_copy_result(st, {out->account_first, out->account_keys32, out->account_body_off, out->account_bodies, out->served_first,
                               out->slot_first, out->slot_keys32, out->slot_body_off, out->slot_bodies, out->proof_first, out->node_index,
                               out->nodes, out->node_off}, [&]() -> int {
        RC(copy_node_set(st, out->node_off, out->nodes));
        if (n + m == 0) {
            out->account_first[0] = out->account_body_off[0] = out->served_first[0] = out->slot_first[0] = out->slot_body_off[0] = 0;
            out->proof_first[0] = 0;
            return PHANT_GPU_OK;
        }
        Carve c{(uint8_t*)st->snp_res.ptr};
        SnpRes o;
        o.take(c, n, m, ea, st->snp_ab, ns, es, st->snp_sb, st->snp_refs);
        RC(copy_out(ctx, out->account_first, o.afirst, 8ull * (n + 1)));
        RC(copy_out(ctx, out->account_keys32, o.akeys, 32 * ea));
        RC(copy_out(ctx, out->account_body_off, o.aoff, 8 * (ea + 1)));
        RC(copy_out(ctx, out->account_bodies, o.abodies, st->snp_ab));
        RC(copy_out(ctx, out->served_first, o.sfirst, 8ull * (m + 1)));
        RC(copy_out(ctx, out->slot_first, o.slot_first, 8 * (ns + 1)));
        RC(copy_out(ctx, out->slot_keys32, o.skeys, 32 * es));
        RC(copy_out(ctx, out->slot_body_off, o.soff, 8 * (es + 1)));
        RC(copy_out(ctx, out->slot_bodies, o.sbodies, st->snp_sb));
        RC(copy_out(ctx, out->proof_first, o.pfirst, 8ull * (n + m + 1)));
        return copy_out(ctx, out->node_index, o.node_index, 8 * st->snp_refs);
    });
}

// ------------------------------------------------------------------------------------------------
// Resident world state: account and slot reads (phant_gpu_resident_state_read), at the current root or at any root the undo
// journal reaches.  DESIGN.md §4.3g.  One thread per requested key (resident_read.cuh): a binary search in the account trie's
// row table and P's account decoder, or a binary search in the slot table; at a past root first a walk over the window's undo
// records, oldest first, whose device pointers the host uploads as one small table.  No sort, no hashing: at most two
// launches and one synchronisation, whatever the request's size or `back`.  Nothing resident is written and a held witness or
// proof result stays held.
// ------------------------------------------------------------------------------------------------
namespace {

struct RdOut {
    uint8_t *astatus, *bal, *sroot, *code, *sstatus, *svals;
    uint64_t* nonce;
    uint32_t* bad; // an account body that does not decode
};

__global__ void rd_account_kernel(const uint8_t* __restrict__ keys, uint32_t na, const tn::RdRec* __restrict__ recs, uint32_t back,
                                  const KRow* __restrict__ krows, uint32_t n, const uint8_t* __restrict__ arena, RdOut o)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) {
        const tn::RdAccount a = tn::rd_account(recs, back, krows, n, arena, keys + 32ull * i);
        const bool ok = a.status == tn::RD_PRESENT;
        if (a.status == tn::RD_BAD) *o.bad = 1;
        o.astatus[i] = (uint8_t)a.status;
        o.nonce[i] = ok ? a.nonce : 0;
        for (uint32_t b = 0; b < 32; ++b) {
            o.bal[32ull * i + b] = ok && b >= 32 - a.bal_len ? a.bal[b - (32 - a.bal_len)] : 0;
            o.sroot[32ull * i + b] = ok ? a.sroot[b] : 0;
            o.code[32ull * i + b] = ok ? a.code[b] : 0;
        }
    }
}

__global__ void rd_slot_kernel(const uint8_t* __restrict__ akeys, const uint32_t* __restrict__ sacc, const uint8_t* __restrict__ skeys, uint32_t ms,
                               const tn::RdRec* __restrict__ recs, uint32_t back, const SlotRow* __restrict__ S, uint32_t nS, RdOut o)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < ms; j += gridDim.x * blockDim.x) {
        const tn::RdSlot v = tn::rd_slot(recs, back, S, nS, akeys + 32ull * sacc[j], skeys + 32ull * j);
        o.sstatus[j] = (uint8_t)v.status;
        for (uint32_t b = 0; b < 32; ++b) o.svals[32ull * j + b] = v.status == tn::RD_PRESENT ? v.val[b] : 0;
    }
}

// The state at `back` (0: the current one; back <= the journal's size): the window's undo records, the last `back`, oldest
// first, where they lie on the device (RsDiff, then the old storage roots), copied into `table` (`back` entries the caller
// carved; null: no kernel reads them) and counted in h2d_bytes; `root` (nullable) receives the root at `back`.
int rs_window(phant_gpu_resident_state* st, uint32_t back, tn::RdRec* table, uint8_t* root)
{
    phant_gpu_ctx* ctx = st->ctx;
    const uint64_t first = st->journal.size() - back;
    if (root) memcpy(root, back ? st->journal[first].root : st->acct_sp.root, 32);
    if (!table || !back) return PHANT_GPU_OK;
    std::vector<tn::RdRec> recs(back);
    for (uint32_t k = 0; k < back; ++k) {
        const phant_gpu_resident_state::Record& r = st->journal[first + k];
        Carve c{(uint8_t*)r.buf.ptr};
        RsDiff d;
        d.take(c, r.na, r.ms);
        const uint8_t* sroot = c.take<uint8_t>(32ull * r.na);
        recs[k] = tn::RdRec{d.akeys, d.aflags, d.nonce, d.bal, d.code, sroot, d.sacc, d.skeys, d.svals, r.na, r.ms};
    }
    CU(cudaMemcpyAsync(table, recs.data(), sizeof(tn::RdRec) * back, cudaMemcpyHostToDevice, ctx->stream));
    ctx->stats.h2d_bytes += sizeof(tn::RdRec) * back;
    return PHANT_GPU_OK;
}

int rs_read(phant_gpu_resident_state* st, const phant_gpu_proof_request* q, uint32_t back, phant_gpu_state_read_values* out,
            uint8_t out_root[32])
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    RC(check_request_host(ctx, q));
    if (back > st->journal.size()) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({out->account_status, out->nonce, out->balance32, out->storage_root32, out->code_hash32, out->slot_status, out->slot_vals32,
                    out_root}))
        return PHANT_GPU_E_INVALID; // host pointers, as the request
    const uint32_t na = (uint32_t)q->n_accounts, ms = (uint32_t)q->n_slots;
    if (na == 0) return rs_window(st, back, nullptr, out_root); // no key (a slot needs an account)

    // ---- keys and descriptors in, one launch per key kind, requested outputs out ----
    uint8_t *akeys, *skeys;
    uint32_t* sacc;
    tn::RdRec* drecs;
    RdOut o;
    RC(carve(ctx, st->in, [&](Carve& c) {
        akeys = c.take<uint8_t>(32ull * na); sacc = c.take<uint32_t>(ms); skeys = c.take<uint8_t>(32ull * ms); drecs = c.take<tn::RdRec>(back);
        o.astatus = c.take<uint8_t>(na); o.nonce = c.take<uint64_t>(na); o.bal = c.take<uint8_t>(32ull * na); o.sroot = c.take<uint8_t>(32ull * na);
        o.code = c.take<uint8_t>(32ull * na); o.sstatus = c.take<uint8_t>(ms); o.svals = c.take<uint8_t>(32ull * ms); o.bad = c.take<uint32_t>(1);
    }));
    RC(stage_request(ctx, q, akeys, sacc, skeys));
    RC(rs_window(st, back, drecs, out_root));
    CU(cudaMemsetAsync(o.bad, 0, 4, s));
    rd_account_kernel<<<grid1d(dev, na, 128), 128, 0, s>>>(akeys, na, drecs, back, st->acct_rows(), (uint32_t)st->acct_sp.n, st->acct_arena(), o);
    ctx->stats.launches++;
    if (ms) {
        rd_slot_kernel<<<grid1d(dev, ms, 128), 128, 0, s>>>(akeys, sacc, skeys, ms, drecs, back, st->slot_table(), st->nS, o);
        ctx->stats.launches++;
    }
    RC(copy_out(ctx, out->account_status, o.astatus, na));
    RC(copy_out(ctx, out->nonce, o.nonce, 8ull * na));
    RC(copy_out(ctx, out->balance32, o.bal, 32ull * na));
    RC(copy_out(ctx, out->storage_root32, o.sroot, 32ull * na));
    RC(copy_out(ctx, out->code_hash32, o.code, 32ull * na));
    RC(copy_out(ctx, out->slot_status, o.sstatus, ms));
    RC(copy_out(ctx, out->slot_vals32, o.svals, 32ull * ms));
    uint32_t bad = 0;
    RC(copy_out(ctx, &bad, o.bad, 4));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    return bad ? rs_undecodable_leaf(ctx) : PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_resident_state_read(phant_gpu_resident_state* st, const phant_gpu_proof_request* req, uint32_t back,
                                             phant_gpu_state_read_values* out, uint8_t out_root[32])
{
    if (!req || !out || !out_root) return PHANT_GPU_E_INVALID;
    RC(rs_enter(st));
    return rs_read(st, req, back, out, out_root);
}

// ------------------------------------------------------------------------------------------------
// Resident world state: account and storage ranges (phant_gpu_resident_state_range), at the current root or at any root the
// undo journal reaches.  DESIGN.md §4.3h.  Per range (resident_range.cuh): two binary searches in the current table and two
// in each of the window's records give its candidate parts; at a past root the candidates are gathered, sorted by (range,
// key), deduplicated and resolved with read's per-key rules, and the present ones ranked.  With no record the current
// table's run is the answer as it is.  Then one scan of the entries per range, one read-back, one fill.  No hashing; the
// launches do not grow with the number of ranges, `back` or the entries returned.  Nothing resident is written and a held
// witness or proof result stays held.
// ------------------------------------------------------------------------------------------------
namespace {

// the ranges of one call: r < n is account range r, r >= n storage range r - n
struct RgRanges {
    const uint8_t *origin, *limit, *sacct; // (n + m) x 32, (n + m) x 32, m x 32
    const uint32_t* max;                   // n + m
    uint32_t n, m;
};
// the state at the call's root: the window's records (oldest first) and the current tables
struct RgState {
    const tn::RdRec* recs;
    uint32_t back;
    const KRow* krows;
    uint32_t nK;
    const uint8_t* arena;
    const SlotRow* S;
    uint32_t nS;
};
struct RgOut {
    uint8_t *akeys, *bal, *sroot, *code, *skeys, *svals;
    uint64_t* nonce;
    uint32_t* bad; // an account body that does not decode
};

// the back + 1 candidate parts of every range
__global__ void rg_parts_kernel(RgRanges q, RgState t, uint32_t* __restrict__ lo, uint64_t* __restrict__ cnt)
{
    const uint64_t P = t.back + 1;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < q.n + q.m; r += gridDim.x * blockDim.x) {
        const uint8_t *o = q.origin + 32ull * r, *l = q.limit + 32ull * r;
        if (r < q.n) tn::rg_account_parts(t.recs, t.back, t.krows, t.nK, o, l, q.max[r], lo + P * r, cnt + P * r);
        else tn::rg_slot_parts(t.recs, t.back, t.S, t.nS, q.sacct + 32ull * (r - q.n), o, l, q.max[r], lo + P * r, cnt + P * r);
    }
}

// candidate j (part offsets poff over (n + m)(back + 1) parts): its key and range
__global__ void rg_cand_kernel(RgRanges q, RgState t, const uint32_t* __restrict__ lo, const uint64_t* __restrict__ poff, uint64_t C,
                               uint8_t* __restrict__ ckeys, uint32_t* __restrict__ cseg)
{
    const uint64_t P = t.back + 1, parts = P * (q.n + q.m);
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < C; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t pp = tn::rg_segment(poff, parts, j);
        const uint32_t r = (uint32_t)(pp / P), p = (uint32_t)(pp % P);
        const uint8_t* k = r < q.n ? tn::rg_account_key(t.recs, t.krows, p, lo[pp], j - poff[pp]) : tn::rg_slot_key(t.recs, t.S, p, lo[pp], j - poff[pp]);
        for (int b = 0; b < 32; ++b) ckeys[32 * j + b] = k[b];
        cseg[j] = r;
    }
}

// sorted candidate j: 1 when it is present at the root and not the same key as its predecessor in the same range
__global__ void rg_resolve_kernel(RgRanges q, RgState t, const uint8_t* __restrict__ ckeys, const uint32_t* __restrict__ cseg,
                                  const uint32_t* __restrict__ perm, uint64_t C, uint64_t* __restrict__ pres, uint32_t* __restrict__ bad)
{
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < C; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t i = perm[j], r = cseg[i];
        const uint8_t* key = ckeys + 32ull * i;
        if (j && cseg[perm[j - 1]] == r && tn::rd_cmp32(ckeys + 32ull * perm[j - 1], key) == 0) { pres[j] = 0; continue; }
        uint32_t status;
        if (r < q.n) status = tn::rd_account(t.recs, t.back, t.krows, t.nK, t.arena, key).status;
        else status = tn::rd_slot(t.recs, t.back, t.S, t.nS, q.sacct + 32ull * (r - q.n), key).status;
        if (status == tn::RD_BAD) *bad = 1;
        pres[j] = status == tn::RD_PRESENT;
    }
}

// entries and `more` per range: present keys counted by the scan x of the sorted candidates, or (no record) part 0 as it is
__global__ void rg_count_kernel(RgRanges q, uint32_t back, const uint64_t* __restrict__ cnt, const uint64_t* __restrict__ poff,
                                const uint64_t* __restrict__ x, uint64_t* __restrict__ ent, uint8_t* __restrict__ more)
{
    const uint64_t P = back + 1;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < q.n + q.m; r += gridDim.x * blockDim.x) {
        const uint64_t present = back ? x[poff[P * (r + 1)]] - x[poff[P * r]] : cnt[r];
        tn::rg_select(present, q.max[r], ent[r], more[r]);
    }
}

// entry e (offsets E over the n + m ranges; account entries first): its key and value
__global__ void rg_fill_kernel(RgRanges q, RgState t, const uint32_t* __restrict__ lo, const uint64_t* __restrict__ poff,
                               const uint64_t* __restrict__ x, const uint8_t* __restrict__ ckeys, const uint32_t* __restrict__ perm,
                               const uint64_t* __restrict__ E, uint64_t total, RgOut o)
{
    const uint64_t P = t.back + 1;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)tn::rg_segment(E, q.n + q.m, e);
        const uint64_t at = e - E[r];
        const uint8_t* key;
        if (t.back) key = ckeys + 32ull * perm[tn::rg_nth_present(x, poff[P * r], poff[P * (r + 1)], at)];
        else key = r < q.n ? tn::rg_account_key(t.recs, t.krows, 0, lo[r], at) : tn::rg_slot_key(t.recs, t.S, 0, lo[r], at);
        if (r < q.n) {
            const tn::RdAccount a = tn::rd_account(t.recs, t.back, t.krows, t.nK, t.arena, key);
            if (a.status != tn::RD_PRESENT) { *o.bad = 1; continue; }
            o.nonce[e] = a.nonce;
            for (uint32_t b = 0; b < 32; ++b) {
                o.akeys[32 * e + b] = key[b];
                o.bal[32 * e + b] = b >= 32 - a.bal_len ? a.bal[b - (32 - a.bal_len)] : 0;
                o.sroot[32 * e + b] = a.sroot[b];
                o.code[32 * e + b] = a.code[b];
            }
        } else {
            const uint64_t s = e - E[q.n];
            const tn::RdSlot v = tn::rd_slot(t.recs, t.back, t.S, t.nS, q.sacct + 32ull * (r - q.n), key);
            if (v.status != tn::RD_PRESENT) { *o.bad = 1; continue; }
            for (uint32_t b = 0; b < 32; ++b) {
                o.skeys[32 * s + b] = key[b];
                o.svals[32 * s + b] = v.val[b];
            }
        }
    }
}

int rs_range(phant_gpu_resident_state* st, const phant_gpu_range_request* q, uint32_t back, phant_gpu_range_values* out,
             uint8_t out_root[32])
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint64_t n64 = q->n_account_ranges, m64 = q->n_storage_ranges;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // host pointers only, as read
    if (n64 > (1ull << 28) || m64 > (1ull << 28)) return PHANT_GPU_E_INVALID;
    if (n64 && (!q->account_origin32 || !q->account_limit32 || !q->account_max)) return PHANT_GPU_E_INVALID;
    if (m64 && (!q->storage_account32 || !q->storage_origin32 || !q->storage_limit32 || !q->storage_max)) return PHANT_GPU_E_INVALID;
    if (back > st->journal.size()) return PHANT_GPU_E_INVALID;
    if (!host_ptrs({q->account_origin32, q->account_limit32, q->account_max, q->storage_account32, q->storage_origin32, q->storage_limit32,
                    q->storage_max, out->account_first, out->account_more, out->account_keys32, out->nonce, out->balance32, out->storage_root32,
                    out->code_hash32, out->slot_first, out->slot_more, out->slot_keys32, out->slot_vals32, out_root}))
        return PHANT_GPU_E_INVALID;
    uint64_t sum_a = 0, sum_s = 0;
    for (uint64_t r = 0; r < n64; ++r) sum_a += q->account_max[r];
    for (uint64_t r = 0; r < m64; ++r) sum_s += q->storage_max[r];
    if (sum_a >= (1ull << 32) || sum_s >= (1ull << 32)) return PHANT_GPU_E_INVALID;
    const uint32_t n = (uint32_t)n64, m = (uint32_t)m64, nr = n + m;
    const uint64_t P = back + 1, parts = P * nr;

    // ---- ranges and record descriptors in; the parts of every range ----
    RgRanges g{nullptr, nullptr, nullptr, nullptr, n, m};
    uint8_t *origin, *limit, *sacct, *more;
    uint32_t *max, *lo, *bad;
    uint64_t *cnt, *poff, *ent, *E;
    tn::RdRec* drecs;
    RC(carve(ctx, st->in, [&](Carve& c) {
        origin = c.take<uint8_t>(32ull * nr); limit = c.take<uint8_t>(32ull * nr); sacct = c.take<uint8_t>(32ull * m); max = c.take<uint32_t>(nr);
        drecs = c.take<tn::RdRec>(back); lo = c.take<uint32_t>(parts); cnt = c.take<uint64_t>(parts + 1); poff = c.take<uint64_t>(parts + 1);
        ent = c.take<uint64_t>(nr + 1); E = c.take<uint64_t>(nr + 1); more = c.take<uint8_t>(nr); bad = c.take<uint32_t>(1);
    }));
    g.origin = origin; g.limit = limit; g.sacct = sacct; g.max = max;
    RC(rs_window(st, back, drecs, out_root));
    const RgState t{drecs, back, st->acct_rows(), (uint32_t)st->acct_sp.n, st->acct_arena(), st->slot_table(), st->nS};
    if (n) {
        CU(cudaMemcpyAsync(origin, q->account_origin32, 32ull * n, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(limit, q->account_limit32, 32ull * n, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(max, q->account_max, 4ull * n, cudaMemcpyHostToDevice, s));
    }
    if (m) {
        CU(cudaMemcpyAsync(origin + 32ull * n, q->storage_origin32, 32ull * m, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(limit + 32ull * n, q->storage_limit32, 32ull * m, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(max + n, q->storage_max, 4ull * m, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(sacct, q->storage_account32, 32ull * m, cudaMemcpyHostToDevice, s));
    }
    ctx->stats.h2d_bytes += 68ull * nr + 32ull * m;
    CU(cudaMemsetAsync(bad, 0, 4, s));
    if (nr) {
        rg_parts_kernel<<<grid1d(dev, nr, 128), 128, 0, s>>>(g, t, lo, cnt);
        ctx->stats.launches++;
    }

    // ---- at a past root: the candidates, sorted by (range, key), deduplicated, resolved and ranked ----
    uint8_t* ckeys = nullptr;
    uint32_t* perm = nullptr;
    uint64_t* x = nullptr;
    if (back) {
        RC(scan_sizes(ctx, cnt, poff, parts));
        uint64_t C = 0;
        RC(copy_out(ctx, &C, poff + parts, 8));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches++;
        if (C >= (1ull << 32)) {
            snprintf(ctx->last_error, sizeof ctx->last_error, "resident state range: %llu candidates, more than one sort holds",
                     (unsigned long long)C);
            return PHANT_GPU_E_OOM;
        }
        uint32_t* cseg;
        uint64_t* pres;
        RC(carve(ctx, st->dirty, [&](Carve& c) {
            ckeys = c.take<uint8_t>(32 * C); cseg = c.take<uint32_t>(C); perm = c.take<uint32_t>(C); pres = c.take<uint64_t>(C + 1);
            x = c.take<uint64_t>(C + 1);
        }));
        if (C) {
            rg_cand_kernel<<<grid1d(dev, C, 256), 256, 0, s>>>(g, t, lo, poff, C, ckeys, cseg);
            RC(sort_by_segment_and_hash(ctx, ckeys, cseg, (uint32_t)C, perm, st->sort));
            rg_resolve_kernel<<<grid1d(dev, C, 128), 128, 0, s>>>(g, t, ckeys, cseg, perm, C, pres, bad);
            ctx->stats.launches += 2;
        }
        RC(scan_sizes(ctx, pres, x, C));
        ctx->stats.launches++;
    }

    // ---- entries per range, their offsets, one read-back ----
    std::vector<uint64_t> hE(nr + 1, 0);
    if (nr) {
        rg_count_kernel<<<grid1d(dev, nr, 256), 256, 0, s>>>(g, back, cnt, poff, x, ent, more);
        RC(scan_sizes(ctx, ent, E, nr));
        RC(copy_out(ctx, hE.data(), E, 8ull * (nr + 1)));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches += 2;
    }
    const uint64_t ea = hE[n], es = hE[nr] - hE[n];

    // ---- the entries, then everything requested out ----
    RgOut o;
    RC(carve(ctx, st->work, [&](Carve& c) {
        o.akeys = c.take<uint8_t>(32 * ea); o.nonce = c.take<uint64_t>(ea); o.bal = c.take<uint8_t>(32 * ea); o.sroot = c.take<uint8_t>(32 * ea);
        o.code = c.take<uint8_t>(32 * ea); o.skeys = c.take<uint8_t>(32 * es); o.svals = c.take<uint8_t>(32 * es);
    }));
    o.bad = bad;
    if (ea + es) {
        rg_fill_kernel<<<grid1d(dev, ea + es, 128), 128, 0, s>>>(g, t, lo, poff, x, ckeys, perm, E, ea + es, o);
        ctx->stats.launches++;
    }
    RC(copy_out(ctx, out->account_more, more, n));
    RC(copy_out(ctx, out->slot_more, more + n, m));
    RC(copy_out(ctx, out->account_keys32, o.akeys, 32 * ea));
    RC(copy_out(ctx, out->nonce, o.nonce, 8 * ea));
    RC(copy_out(ctx, out->balance32, o.bal, 32 * ea));
    RC(copy_out(ctx, out->storage_root32, o.sroot, 32 * ea));
    RC(copy_out(ctx, out->code_hash32, o.code, 32 * ea));
    RC(copy_out(ctx, out->slot_keys32, o.skeys, 32 * es));
    RC(copy_out(ctx, out->slot_vals32, o.svals, 32 * es));
    uint32_t hbad = 0;
    RC(copy_out(ctx, &hbad, bad, 4));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (hbad) return rs_undecodable_leaf(ctx);
    if (out->account_first)
        for (uint32_t r = 0; r <= n; ++r) out->account_first[r] = hE[r];
    if (out->slot_first)
        for (uint32_t r = 0; r <= m; ++r) out->slot_first[r] = hE[n + r] - hE[n];
    return PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_resident_state_range(phant_gpu_resident_state* st, const phant_gpu_range_request* req, uint32_t back,
                                              phant_gpu_range_values* out, uint8_t out_root[32])
{
    if (!req || !out || !out_root) return PHANT_GPU_E_INVALID;
    RC(rs_enter(st));
    return rs_range(st, req, back, out, out_root);
}

// ------------------------------------------------------------------------------------------------
// Resident world state: contract code (phant_gpu_resident_state_put_codes / _codes / _prune_codes).  DESIGN.md §4.3i.
// A row table sorted by codeHash (KRow: key = keccak(code), off / len into a code arena of 16-byte aligned entries), ping-pong
// across merges like kind 1's.  put hashes the codes with K, sorts them with the apply's sort, flags repeats and the empty
// code, classifies the rest against the table with the apply's classifier, appends the new codes to the arena and merges.
// codes is one binary search per hash (resident_code.cuh), a scan, one read-back and a gather.  prune marks the codes that
// the current account rows and the window's undo records name, then gathers the kept rows and bytes into a fresh table and
// arena.  No launch count depends on how many codes, hashes, accounts or records a call sees.  Nothing else resident is
// written, and the three calls stay out of apply, revert, witness, prove, read and range.
// ------------------------------------------------------------------------------------------------
namespace rs_body {
#include "resident_code.cuh"
}
namespace {

// put: sorted row j is code perm[j]: its key and length, where it lies in the staged bytes, and `skip` when it repeats row
// j - 1 or is the empty code (never stored)
__global__ void cd_rows_kernel(const uint8_t* __restrict__ hashes, const uint64_t* __restrict__ off, const uint32_t* __restrict__ perm, uint32_t m,
                               KRow* __restrict__ rows, SRec* __restrict__ src, uint8_t* __restrict__ skip)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint32_t i = perm[j];
        KRow& r = rows[j];
        const uint4* h = reinterpret_cast<const uint4*>(hashes + 32ull * i);
        uint4* k = reinterpret_cast<uint4*>(r.key);
        k[0] = h[0]; k[1] = h[1];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);
        r.off = 0;
        r.len = len;
        r.cache[0] = 0;
        src[j] = SRec{off[i], len, 0};
        skip[j] = len == 0 || (j && cmp_key32(hashes + 32ull * perm[j - 1], hashes + 32ull * i) == 0);
    }
}
// arena bytes (16-byte aligned) of each row the classifier found new; counters64[0] += the new codes' own lengths
__global__ void cd_size_kernel(const KRow* __restrict__ rows, const uint8_t* __restrict__ kind, uint32_t m, uint64_t* __restrict__ size,
                               unsigned long long* __restrict__ counters64)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const bool ins = kind[j] == 2;
        size[j] = ins ? (rows[j].len + 15ull) & ~15ull : 0;
        if (ins) atomicAdd(counters64, (unsigned long long)rows[j].len);
    }
}
// each new row's place in the arena (base + its offset among the new codes); rows that are not new copy nothing
__global__ void cd_place_kernel(KRow* __restrict__ rows, SRec* __restrict__ src, const uint8_t* __restrict__ kind, const uint64_t* __restrict__ ioff,
                                uint32_t m, uint64_t base)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        rows[j].off = base + ioff[j];
        if (kind[j] != 2) src[j].len = 0;
    }
}

// codes: per hash its status, arena slice and length
__global__ void cd_lookup_kernel(const KRow* __restrict__ rows, uint32_t n, const uint8_t* __restrict__ hashes, uint32_t m, uint8_t* __restrict__ status,
                                 SRec* __restrict__ rec, uint64_t* __restrict__ size)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const tn::CdCode c = tn::cd_lookup(rows, n, hashes + 32ull * i);
        status[i] = (uint8_t)c.status;
        rec[i] = SRec{c.off, c.len, 0};
        size[i] = c.len;
    }
}

// prune: the codes the current account rows name; *bad when a body does not decode
__global__ void cd_mark_accounts_kernel(const KRow* __restrict__ krows, uint32_t nK, const uint8_t* __restrict__ arena, const KRow* __restrict__ rows,
                                        uint32_t n, uint8_t* __restrict__ keep, uint32_t* __restrict__ bad)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nK; i += gridDim.x * blockDim.x) {
        const uint8_t* h = tn::cd_account_code(krows, i, arena);
        if (!h) { *bad = 1; continue; }
        tn::cd_mark(rows, n, h, keep);
    }
}
// the codes the window's records name: record blockIdx.y, its entries across blockIdx.x
__global__ void cd_mark_records_kernel(const tn::RdRec* __restrict__ recs, const KRow* __restrict__ rows, uint32_t n, uint8_t* __restrict__ keep)
{
    const tn::RdRec& R = recs[blockIdx.y];
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < R.na; p += gridDim.x * blockDim.x) tn::cd_mark(rows, n, tn::cd_record_code(R, p), keep);
}
// kept rows: flag, arena bytes (16-byte aligned); counters64[0] += their codes' own lengths
__global__ void cd_keep_kernel(const KRow* __restrict__ rows, const uint8_t* __restrict__ keep, uint32_t n, uint32_t* __restrict__ flag,
                               uint64_t* __restrict__ size, unsigned long long* __restrict__ counters64)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        flag[i] = keep[i];
        size[i] = keep[i] ? (rows[i].len + 15ull) & ~15ull : 0;
        if (keep[i]) atomicAdd(counters64, (unsigned long long)rows[i].len);
    }
}
// kept row i -> fresh row idx[i] at arena offset off[i], with where its bytes lie now
__global__ void cd_compact_kernel(const KRow* __restrict__ rows, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ idx,
                                  const uint64_t* __restrict__ off, uint32_t n, KRow* __restrict__ fresh, SRec* __restrict__ src,
                                  uint64_t* __restrict__ dst)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (!flag[i]) continue;
        const uint32_t q = idx[i];
        KRow r = rows[i];
        src[q] = SRec{r.off, r.len, 0};
        dst[q] = off[i];
        r.off = off[i];
        fresh[q] = r;
    }
}

int cd_put(phant_gpu_resident_state* st, const uint8_t* codes, const uint64_t* code_off, uint64_t n64, uint8_t* hashes32)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    if (n64 >= (1ull << 28) || (n64 && !code_off)) return PHANT_GPU_E_INVALID;
    if ((ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) || !host_ptrs({codes, code_off, hashes32})) return PHANT_GPU_E_INVALID;
    if (n64 == 0) return PHANT_GPU_OK;
    const uint32_t m = (uint32_t)n64;
    for (uint32_t i = 0; i < m; ++i)
        if (code_off[i + 1] < code_off[i] || code_off[i + 1] - code_off[i] > 0xffffffffull) return PHANT_GPU_E_INVALID;
    const uint64_t total = code_off[m] - code_off[0];
    if (total && !codes) return PHANT_GPU_E_INVALID;
    std::vector<uint64_t> rel(m + 1);
    for (uint32_t i = 0; i <= m; ++i) rel[i] = code_off[i] - code_off[0];
    const uint32_t n = st->n_codes;

    // ---- the codes in, hashed, sorted into rows, classified against the table ----
    uint8_t *bytes, *hashes, *skip, *kind;
    uint64_t *off, *size, *ioff;
    uint32_t *perm, *lb, *ins_flag, *ins_index, *del_flag, *ins_at, *keep, *K, *I, *counters;
    KRow* rows;
    SRec* src;
    RC(carve(ctx, st->in, [&](Carve& c) { bytes = c.take<uint8_t>(total + 64); off = c.take<uint64_t>(m + 1); hashes = c.take<uint8_t>(32ull * m); }));
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        perm = c.take<uint32_t>(m); rows = c.take<KRow>(m); src = c.take<SRec>(m); skip = c.take<uint8_t>(m); kind = c.take<uint8_t>(m);
        lb = c.take<uint32_t>(m); ins_flag = c.take<uint32_t>(m + 1); ins_index = c.take<uint32_t>(m + 1); size = c.take<uint64_t>(m + 1);
        ioff = c.take<uint64_t>(m + 1); counters = c.take<uint32_t>(16);
        del_flag = c.take<uint32_t>((n + 3ull) * 5); // del_flag and ins_at first: one memset clears both
    }));
    ins_at = del_flag + n + 3; keep = ins_at + n + 3; K = keep + n + 3; I = K + n + 3;
    if (total) CU(cudaMemcpyAsync(bytes, codes + code_off[0], total, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(off, rel.data(), 8ull * (m + 1), cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += total + 8ull * (m + 1);
    RC(ctx->hash_csr(bytes, off, m, total, hashes));
    RC(sort_by_segment_and_hash(ctx, hashes, nullptr, m, perm, st->sort));
    CU(cudaMemsetAsync(counters, 0, 64, s));
    CU(cudaMemsetAsync(del_flag, 0, 4ull * (n + 3) * 2, s));
    const KRow* table = (const KRow*)st->code_rows[st->cc].ptr;
    cd_rows_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(hashes, off, perm, m, rows, src, skip);
    // a skipped row classifies as a no-op whether or not the table holds its key (skip is both `del` and `absent`)
    rs_classify_kernel<KRow, 32><<<grid1d(dev, m, 128), 128, 0, s>>>(table, n, rows, m, skip, skip, lb, kind, del_flag, ins_at, ins_flag, counters);
    unsigned long long* added = (unsigned long long*)(counters + 8);
    cd_size_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(rows, kind, m, size, added);
    RC(scan_sizes(ctx, size, ioff, m));
    uint32_t hc[16];
    uint64_t grow = 0;
    CU(cudaMemcpyAsync(hc, counters, 64, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&grow, ioff + m, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 4;
    ctx->stats.d2h_bytes += 72;
    const uint32_t n_ins = hc[0];
    uint64_t added_len;
    memcpy(&added_len, hc + 8, 8);

    // ---- new codes to the arena's end, the rows merged into the other table; the store switches only when all is done ----
    if (n_ins) {
        RC(grow_keep(ctx, st->code_arena, st->code_used, st->code_used + grow + 64)); // contents kept: the store is unchanged
        RC(st->code_rows[1 - st->cc].reserve(ctx, sizeof(KRow) * ((uint64_t)n + n_ins) + 64));
        cd_place_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(rows, src, kind, ioff, m, st->code_used);
        st_gather_vals_kernel<SRec><<<grid1d(dev, m, 256, 32), 256, 0, s>>>(bytes, src, ioff, m, (uint8_t*)st->code_arena.ptr + st->code_used);
        ctx->stats.launches += 2;
        int cur = st->cc;
        RC(rs_merge<KRow>(ctx, st->code_rows, cur, n, rows, m, kind, lb, ins_flag, del_flag, ins_at, keep, K, I, ins_index));
    }
    if (hashes32) CU(cudaMemcpyAsync(hashes32, hashes, 32ull * m, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (hashes32) ctx->stats.d2h_bytes += 32ull * m;
    if (n_ins) {
        st->cc = 1 - st->cc;
        st->n_codes = n + n_ins;
        st->code_used += grow;
        st->code_bytes += added_len;
    }
    return PHANT_GPU_OK;
}

int cd_codes(phant_gpu_resident_state* st, const uint8_t* hashes32, uint64_t n64, uint8_t* status, uint64_t* code_off, uint8_t* codes,
             uint64_t codes_cap)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    if (n64 >= (1ull << 28) || !code_off || (n64 && (!hashes32 || !status))) return PHANT_GPU_E_INVALID;
    if ((ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) || !host_ptrs({hashes32, status, code_off, codes})) return PHANT_GPU_E_INVALID;
    code_off[0] = 0;
    if (n64 == 0) return PHANT_GPU_OK;
    const uint32_t m = (uint32_t)n64;

    // ---- one binary search per hash, the lengths scanned, status and offsets out (sync 1) ----
    uint8_t *hashes, *dstatus;
    uint64_t *size, *offs;
    SRec* rec;
    RC(carve(ctx, st->in, [&](Carve& c) {
        hashes = c.take<uint8_t>(32ull * m); dstatus = c.take<uint8_t>(m); rec = c.take<SRec>(m); size = c.take<uint64_t>(m + 1);
        offs = c.take<uint64_t>(m + 1);
    }));
    CU(cudaMemcpyAsync(hashes, hashes32, 32ull * m, cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += 32ull * m;
    cd_lookup_kernel<<<grid1d(dev, m, 128), 128, 0, s>>>((const KRow*)st->code_rows[st->cc].ptr, st->n_codes, hashes, m, dstatus, rec, size);
    RC(scan_sizes(ctx, size, offs, m));
    RC(copy_out(ctx, status, dstatus, m));
    RC(copy_out(ctx, code_off, offs, 8ull * (m + 1)));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    const uint64_t total = code_off[m];
    if (!codes || total > codes_cap || total == 0) return PHANT_GPU_OK;

    // ---- the bytes gathered and copied out (sync 2) ----
    uint8_t* out;
    RC(carve(ctx, st->work, [&](Carve& c) { out = c.take<uint8_t>(total); }));
    st_gather_vals_kernel<SRec><<<grid1d(dev, m, 256, 32), 256, 0, s>>>((const uint8_t*)st->code_arena.ptr, rec, offs, m, out);
    RC(copy_out(ctx, codes, out, total));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    ctx->stats.launches++;
    return PHANT_GPU_OK;
}

// the fresh table and arena of a prune, filled from the marks; on success they replace the store's
int cd_prune_into(phant_gpu_resident_state* st, DevBuf& fresh_arena)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t n = st->n_codes;
    const uint32_t back = (uint32_t)st->journal.size();
    uint32_t max_na = 0;
    for (const phant_gpu_resident_state::Record& r : st->journal) max_na = r.na > max_na ? r.na : max_na;

    // ---- marks: the current account rows, then every record of the window in one launch ----
    uint8_t* keep;
    uint32_t *flag, *idx, *bad;
    uint64_t *size, *off, *dst;
    unsigned long long* kept_len;
    SRec* src;
    tn::RdRec* drecs;
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        keep = c.take<uint8_t>(n); flag = c.take<uint32_t>(n + 1); idx = c.take<uint32_t>(n + 1); size = c.take<uint64_t>(n + 1);
        off = c.take<uint64_t>(n + 1); dst = c.take<uint64_t>(n); src = c.take<SRec>(n); drecs = c.take<tn::RdRec>(back);
        bad = c.take<uint32_t>(4); kept_len = c.take<unsigned long long>(1);
    }));
    const KRow* rows = (const KRow*)st->code_rows[st->cc].ptr;
    const SparseTrie& sp = st->acct_sp;
    CU(cudaMemsetAsync(keep, 0, n, s));
    CU(cudaMemsetAsync(bad, 0, 4, s));
    CU(cudaMemsetAsync(kept_len, 0, 8, s));
    RC(rs_window(st, back, drecs, nullptr));
    if (sp.n) {
        cd_mark_accounts_kernel<<<grid1d(dev, sp.n, 128), 128, 0, s>>>(st->acct_rows(), (uint32_t)sp.n, st->acct_arena(), rows, n, keep, bad);
        ctx->stats.launches++;
    }
    if (max_na) {
        cd_mark_records_kernel<<<dim3(grid1d(dev, max_na, 128) / back + 1, back), 128, 0, s>>>(drecs, rows, n, keep);
        ctx->stats.launches++;
    }

    // ---- kept rows counted and placed (sync 1), then gathered into the fresh table and arena (sync 2) ----
    cd_keep_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(rows, keep, n, flag, size, kept_len);
    RC(scan_u32(ctx, flag, idx, n + 1));
    RC(scan_sizes(ctx, size, off, n));
    uint32_t hk[2] = {0, 0};
    uint64_t hb[2] = {0, 0};
    CU(cudaMemcpyAsync(&hk[0], idx + n, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&hk[1], bad, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&hb[0], off + n, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&hb[1], kept_len, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 3;
    ctx->stats.d2h_bytes += 24;
    if (hk[1]) return rs_undecodable_leaf(ctx);
    const uint32_t kept = hk[0];
    const uint64_t bytes = hb[0];
    DevBuf& fresh_rows = st->code_rows[1 - st->cc];
    RC(fresh_rows.reserve(ctx, sizeof(KRow) * (uint64_t)kept + 64));
    RC(fresh_arena.reserve(ctx, bytes + 64));
    cd_compact_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(rows, flag, idx, off, n, (KRow*)fresh_rows.ptr, src, dst);
    st_gather_vals_kernel<SRec><<<grid1d(dev, kept, 256, 32), 256, 0, s>>>((const uint8_t*)st->code_arena.ptr, src, dst, kept, (uint8_t*)fresh_arena.ptr);
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    ctx->stats.launches += 2;
    st->code_arena.release();
    st->code_arena = fresh_arena;
    st->cc = 1 - st->cc;
    st->n_codes = kept;
    st->code_used = bytes;
    st->code_bytes = hb[1];
    return PHANT_GPU_OK;
}

} // namespace

extern "C" int phant_gpu_resident_state_put_codes(phant_gpu_resident_state* st, const uint8_t* codes, const uint64_t* code_off, uint64_t n_codes,
                                                  uint8_t* hashes32)
{
    RC(rs_enter(st));
    return cd_put(st, codes, code_off, n_codes, hashes32);
}

extern "C" int phant_gpu_resident_state_codes(phant_gpu_resident_state* st, const uint8_t* hashes32, uint64_t n, uint8_t* status, uint64_t* code_off,
                                              uint8_t* codes, uint64_t codes_cap)
{
    RC(rs_enter(st));
    return cd_codes(st, hashes32, n, status, code_off, codes, codes_cap);
}

extern "C" int phant_gpu_resident_state_prune_codes(phant_gpu_resident_state* st)
{
    RC(rs_enter(st));
    if (st->n_codes == 0) return PHANT_GPU_OK;
    DevBuf fresh;
    const int rc = cd_prune_into(st, fresh);
    if (rc) fresh.release(); // the store keeps its table and arena
    return rc;
}
