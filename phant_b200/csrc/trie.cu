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

// exclusive scan of cnt u64 sizes into cnt+1 offsets (in[cnt] must be readable; it is forced to 0 first)
int scan_sizes(phant_gpu_ctx* ctx, uint64_t* sizes, uint64_t* offs, uint64_t cnt)
{
    CU(cudaMemsetAsync(sizes + cnt, 0, 8, ctx->stream));
    size_t temp = 0;
    CU(cub::DeviceScan::ExclusiveSum(nullptr, temp, (const uint64_t*)sizes, offs, (int64_t)(cnt + 1), ctx->stream));
    RC(ctx->d_cub.reserve(ctx, temp));
    CU(cub::DeviceScan::ExclusiveSum(ctx->d_cub.ptr, temp, (const uint64_t*)sizes, offs, (int64_t)(cnt + 1), ctx->stream));
    return 0;
}

// bump allocation inside one scratch buffer, every array on a 256-byte boundary; without a base it only measures
struct Carve {
    uint8_t* base = nullptr;
    uint64_t used = 0;
    template <class T> T* take(uint64_t count)
    {
        T* r = base ? (T*)(base + used) : nullptr;
        used += (sizeof(T) * count + 255) & ~255ull;
        return r;
    }
};
// one scratch area sized and placed by one declaration: lay(c) takes every array from c and assigns the caller's pointers;
// it runs once to measure, `buf` grows to fit (plus 256 bytes of tail), and it runs again to place
template <class Lay> int carve(phant_gpu_ctx* ctx, DevBuf& buf, Lay&& lay)
{
    Carve m;
    lay(m);
    RC(buf.reserve(ctx, m.used + 256));
    Carve c{(uint8_t*)buf.ptr};
    lay(c);
    return PHANT_GPU_OK;
}

} // namespace

// ------------------------------------------------------------------------------------------------
// forest builder: keys/vals on the device, keys sorted inside each segment; roots = n_seg * 32 bytes (device)
// ------------------------------------------------------------------------------------------------
int phant_gpu_ctx::build_forest(const uint8_t* d_keys, const uint32_t* d_key_off, const uint8_t* d_vals, const uint64_t* d_val_off,
                                uint32_t n, const uint32_t* d_seg_off, uint32_t n_seg, const uint32_t* d_seg_of_key, uint8_t* d_roots,
                                int slots_hint, uint32_t start_depth, const uint8_t* d_leaf_cache, uint8_t* d_leaf_cache_out,
                                const uint32_t* d_seg_start, const ForestExport* xp)
{
    phant_gpu_ctx* ctx = this;
    cudaStream_t s = stream;
    if (n_seg == 0) return PHANT_GPU_OK;
    PhaseTrace trf(s);
    const Keys k{d_keys, d_key_off};
    const Vals vals{d_vals, d_val_off};
    const uint32_t cap = n ? n : 1;

    // tables
    Tables t;
    RC(carve(ctx, d_b0, [&](Carve& c) {
        t.lo = c.take<uint32_t>(cap); t.hi = c.take<uint32_t>(cap); t.ext_from = c.take<uint32_t>(cap); t.depth = c.take<uint32_t>(cap);
        t.child = c.take<uint32_t>(16ull * cap);
        t.has_value = c.take<uint8_t>(cap);
    }));
    RC(carve(ctx, d_b1, [&](Carve& c) {
        t.ext_list = c.take<uint32_t>(cap); t.leaf_start = c.take<uint32_t>(cap); t.seg_root = c.take<uint32_t>(n_seg);
    }));
    RC(carve(ctx, d_b2, [&](Carve& c) {
        t.ref = c.take<uint8_t>(33ull * 2 * cap); t.ref_len = c.take<uint8_t>(2ull * cap); t.top_digest = c.take<uint8_t>(32ull * cap);
    }));
    RC(d_b3.reserve(ctx, 64)); // counters
    uint32_t* counters = (uint32_t*)d_b3.ptr;
    CU(cudaMemsetAsync(counters, 0, 64, s));
    CU(cudaMemsetAsync(t.leaf_start, 0xff, 4ull * cap, s));

    // keys must be strictly sorted inside each segment (mpt.zig:39 asserts)
    if (n) {
        check_sorted_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(k, d_val_off, d_seg_of_key, n, counters + 4);
        stats.launches++;
    }
    init_roots_kernel<<<grid1d(device, n_seg, 256), 256, 0, s>>>(d_seg_off, n_seg, t, counters, start_depth, d_seg_start);
    stats.launches++;
    uint32_t h[8];
    CU(cudaMemcpyAsync(h, counters, 32, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (h[4]) return PHANT_GPU_E_INVALID;
    // layout choice (see "Two arena layouts" below), from what the check kernel saw: slots need no branch values and small leaves
    uint32_t leaf_stride = 0;
    if (slots_hint > 0) leaf_stride = (uint32_t)slots_hint;
    else if (slots_hint < 0 && n && !h[5] && h[6] <= 64 && h[7] <= 3072) {
        const uint32_t st = (h[7] + h[6] + 16 + 15) & ~15u;
        if ((uint64_t)st * n <= (1ull << 31)) leaf_stride = st;
    }

    // ---- top-down: one launch per BFS level, or the whole BFS in one single-CTA launch for small tries ----
    std::vector<uint32_t> level_beg, level_cnt, level_ext;
    uint32_t beg = 0, cnt = h[0];
    if (cnt && leaf_stride && n <= 8192) { // slot layout implies keys <= 64 bytes = 128 nibbles: at most 129 levels
        constexpr uint32_t MAXL = 160;
        RC(d_tmp_b.reserve(ctx, 4 * (2 + 3 * MAXL)));
        uint32_t* d_levels = (uint32_t*)d_tmp_b.ptr;
        bfs_small_kernel<<<1, 1024, 0, s>>>(k, t, cnt, MAXL, d_levels);
        stats.launches++;
        std::vector<uint32_t> hl(2 + 3 * MAXL);
        CU(cudaMemcpyAsync(hl.data(), d_levels, 4 * hl.size(), cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        if (hl[1 + 3 * MAXL] != 0) return PHANT_GPU_E_INVALID;
        for (uint32_t l = 0; l < hl[0]; ++l) { level_beg.push_back(hl[1 + 3 * l]); level_cnt.push_back(hl[2 + 3 * l]); level_ext.push_back(hl[3 + 3 * l]); }
        cnt = 0;
    }
    while (cnt) {
        CU(cudaMemsetAsync(counters + 1, 0, 8, s));
        expand_kernel<<<grid1d(device, cnt, 128, 16), 128, 0, s>>>(k, t, beg, cnt, beg + cnt, counters);
        stats.launches++;
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
    uint64_t* fixed_leaf = nullptr; uint64_t* fixed_branch = nullptr; uint64_t* fixed_ext = nullptr;
    if (slots) {
        uint32_t max_level = 1;
        for (uint32_t c : level_cnt) if (c > max_level) max_level = c;
        RC(carve(ctx, d_scan_a, [&](Carve& c) {
            fixed_leaf = c.take<uint64_t>(n + 2); fixed_branch = c.take<uint64_t>(max_level + 2); fixed_ext = c.take<uint64_t>(max_level + 2);
        }));
        fixed_offsets_kernel<<<grid1d(device, n + 1, 256), 256, 0, s>>>(fixed_leaf, n, leaf_stride);
        fixed_offsets_kernel<<<grid1d(device, max_level + 1, 256), 256, 0, s>>>(fixed_branch, max_level, BRANCH_STRIDE);
        fixed_offsets_kernel<<<grid1d(device, max_level + 1, 256), 256, 0, s>>>(fixed_ext, max_level, EXT_STRIDE);
        stats.launches += 3;
    }

    trf.mark("    forest: check + BFS");
    // ---- leaves: sizes -> offsets -> encode -> hash -> references (only the leaves the cache cannot answer) ----
    uint8_t* leaf_digests = nullptr;
    if (n) {
        RC(d_b6.reserve(ctx, 32ull * n));
        leaf_digests = (uint8_t*)d_b6.ptr;
        uint32_t m = n;                 // leaves to encode
        const uint32_t* ids = nullptr;  // their key indices (nullptr = all, in order)
        if (d_leaf_cache) {
            uint32_t *flag, *pos, *list;
            RC(carve(ctx, d_tmp_a, [&](Carve& c) { flag = c.take<uint32_t>(n + 2); pos = c.take<uint32_t>(n + 2); list = c.take<uint32_t>(n + 2); }));
            leaf_cache_probe_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(t, n, d_leaf_cache, leaf_digests, flag);
            CU(cudaMemsetAsync(flag + n, 0, 4, s));
            size_t temp = 0;
            CU(cub::DeviceScan::ExclusiveSum(nullptr, temp, (const uint32_t*)flag, pos, (int64_t)(n + 1), s));
            RC(d_cub.reserve(ctx, temp));
            CU(cub::DeviceScan::ExclusiveSum(d_cub.ptr, temp, (const uint32_t*)flag, pos, (int64_t)(n + 1), s));
            compact_iota_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(flag, pos, n, list);
            CU(cudaMemcpyAsync(&m, pos + n, 4, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            ids = list;
            stats.launches += 3;
        }
        if (m) {
            uint64_t *sizes, *offs;
            uint8_t* dg; // compact digests when indirect
            RC(carve(ctx, d_b4, [&](Carve& c) { sizes = c.take<uint64_t>(m + 1); offs = c.take<uint64_t>(m + 1); dg = c.take<uint8_t>(32ull * m); }));
            if (!ids) dg = leaf_digests;
            if (!slots) leaf_size_kernel<<<grid1d(device, m, 256), 256, 0, s>>>(k, vals, t, m, sizes, ids);
            uint64_t total = (uint64_t)m * leaf_stride;
            if (slots) offs = fixed_leaf;
            else {
                RC(scan_sizes(ctx, sizes, offs, m));
                CU(cudaMemcpyAsync(&total, offs + m, 8, cudaMemcpyDeviceToHost, s));
                CU(cudaStreamSynchronize(s));
            }
            RC(d_b5.reserve(ctx, total + 64));
            leaf_encode_kernel<<<grid1d(device, m, 256, 32), 256, 0, s>>>(k, vals, t, m, offs, (uint8_t*)d_b5.ptr, slots ? sizes : nullptr, ids);
            stats.launches += slots ? 1 : 2;
            if (slots) RC(hash_slots((const uint8_t*)d_b5.ptr, offs, sizes, m, dg));
            else RC(hash_csr((const uint8_t*)d_b5.ptr, offs, m, total, dg));
            finalize_ref_kernel<<<grid1d(device, m, 256), 256, 0, s>>>(m, ids, 0, offs, slots ? sizes : nullptr, (const uint8_t*)d_b5.ptr, dg, 0, t,
                                                                     ids ? leaf_digests : nullptr);
            stats.launches++;
            if (xp) {
                forest_export_kernel<<<grid1d(device, m, 256), 256, 0, s>>>(k, t, *xp, 0, m, ids, 0, offs, slots ? sizes : nullptr,
                                                                         (const uint8_t*)d_b5.ptr, dg);
                stats.launches++;
            }
        }
        if (d_leaf_cache_out) {
            leaf_cache_store_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(t, n, leaf_digests, d_leaf_cache_out);
            stats.launches++;
        }
    }

    trf.mark("    forest: leaves");
    // ---- units, deepest level first: branch, then the extension above it where there is one ----
    for (int L = (int)level_beg.size() - 1; L >= 0; --L) {
        const uint32_t lb = level_beg[L], lc = level_cnt[L], le = level_ext[L];
        uint64_t *sizes, *scanned;
        RC(carve(ctx, d_b7, [&](Carve& c) { sizes = c.take<uint64_t>(lc + 1); scanned = c.take<uint64_t>(lc + 1); }));
        if (!slots) branch_size_kernel<<<grid1d(device, lc, 128), 128, 0, s>>>(k, vals, t, n, lb, lc, sizes);
        uint64_t total = (uint64_t)lc * BRANCH_STRIDE;
        uint64_t* offs = slots ? fixed_branch : scanned;
        if (!slots) {
            RC(scan_sizes(ctx, sizes, offs, lc));
            CU(cudaMemcpyAsync(&total, offs + lc, 8, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
        }
        RC(d_b8.reserve(ctx, total + 64));
        RC(d_b9.reserve(ctx, 32ull * lc));
        branch_encode_kernel<<<grid1d(device, lc, 256, 32), 256, 0, s>>>(k, vals, t, n, lb, lc, offs, slots ? sizes : nullptr, slots, (uint8_t*)d_b8.ptr);
        stats.launches += slots ? 1 : 2;
        if (slots) RC(hash_slots((const uint8_t*)d_b8.ptr, offs, sizes, lc, (uint8_t*)d_b9.ptr));
        else RC(hash_csr((const uint8_t*)d_b8.ptr, offs, lc, total, (uint8_t*)d_b9.ptr));
        finalize_ref_kernel<<<grid1d(device, lc, 256), 256, 0, s>>>(lc, nullptr, lb, offs, slots ? sizes : nullptr, (const uint8_t*)d_b8.ptr,
                                                                  (const uint8_t*)d_b9.ptr, n, t, t.top_digest);
        stats.launches++;
        if (xp) {
            forest_export_kernel<<<grid1d(device, lc, 256), 256, 0, s>>>(k, t, *xp, 1, lc, nullptr, lb, offs, slots ? sizes : nullptr,
                                                                      (const uint8_t*)d_b8.ptr, (const uint8_t*)d_b9.ptr);
            stats.launches++;
        }
        if (le) {
            const uint32_t* ids = t.ext_list + lb;
            if (!slots) ext_size_kernel<<<grid1d(device, le, 128), 128, 0, s>>>(k, t, n, ids, le, sizes);
            total = (uint64_t)le * EXT_STRIDE;
            offs = slots ? fixed_ext : scanned;
            if (!slots) {
                RC(scan_sizes(ctx, sizes, offs, le));
                CU(cudaMemcpyAsync(&total, offs + le, 8, cudaMemcpyDeviceToHost, s));
                CU(cudaStreamSynchronize(s));
            }
            RC(d_b8.reserve(ctx, total + 64));
            ext_encode_kernel<<<grid1d(device, le, 128), 128, 0, s>>>(k, t, n, ids, le, offs, (uint8_t*)d_b8.ptr, slots ? sizes : nullptr);
            stats.launches += slots ? 1 : 2;
            if (slots) RC(hash_slots((const uint8_t*)d_b8.ptr, offs, sizes, le, (uint8_t*)d_b9.ptr));
            else RC(hash_csr((const uint8_t*)d_b8.ptr, offs, le, total, (uint8_t*)d_b9.ptr));
            finalize_ref_kernel<<<grid1d(device, le, 256), 256, 0, s>>>(le, ids, 0, offs, slots ? sizes : nullptr, (const uint8_t*)d_b8.ptr,
                                                                      (const uint8_t*)d_b9.ptr, n, t, t.top_digest);
            stats.launches++;
            if (xp) {
                forest_export_kernel<<<grid1d(device, le, 256), 256, 0, s>>>(k, t, *xp, 2, le, ids, 0, offs, slots ? sizes : nullptr,
                                                                          (const uint8_t*)d_b8.ptr, (const uint8_t*)d_b9.ptr);
                stats.launches++;
            }
        }
    }
    trf.mark("    forest: units bottom-up");
    gather_roots_kernel<<<grid1d(device, n_seg, 128), 128, 0, s>>>(t, n_seg, leaf_digests, d_roots);
    stats.launches++;
    CU(cudaGetLastError());
    return PHANT_GPU_OK;
}

// ------------------------------------------------------------------------------------------------
// M
// ------------------------------------------------------------------------------------------------
extern "C" int phant_gpu_mpt_root(phant_gpu_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* vals,
                                  const uint64_t* val_off, uint64_t n, uint8_t out_root[32])
{
    if (!ctx || !out_root || (n && (!key_off || !val_off))) return PHANT_GPU_E_INVALID;
    if (n >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    static const uint8_t EMPTY[32] = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                      0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};
    if (n == 0) { memcpy(out_root, EMPTY, 32); return PHANT_GPU_OK; }
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
    RC(ctx->build_forest(d_keys, d_koff, d_vals, d_voff, (uint32_t)n, (const uint32_t*)ctx->d_first.ptr, 1, nullptr, (uint8_t*)ctx->d_roots.ptr,
                         /*layout decided on the device*/ -1));
    CU(cudaMemcpyAsync(out_root, ctx->d_roots.ptr, 32, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += 32;
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
    RC(ctx->build_forest(dk, dko, dv, dvo, (uint32_t)n, dseg, (uint32_t)n_tries, dsok, (uint8_t*)ctx->d_roots.ptr, -1));
    CU(cudaMemcpyAsync(out_roots, ctx->d_roots.ptr, 32 * n_tries, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += 32 * n_tries;
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

} // namespace

// stable LSD radix sort of n items by (segment, 32-byte big-endian hash): perm_out[i] = index of the i-th smallest
int phant_gpu_ctx::sort_by_segment_and_hash(const uint8_t* d_hashes, const uint32_t* d_seg /*nullable*/, uint32_t n, uint32_t* d_perm_out,
                                            DevBuf& scratch)
{
    phant_gpu_ctx* ctx = this;
    cudaStream_t s = stream;
    if (n == 0) return PHANT_GPU_OK;
    uint64_t *kin, *kout;
    uint32_t *pa, *pb, *sk;
    RC(carve(ctx, scratch, [&](Carve& c) {
        kin = c.take<uint64_t>(n); kout = c.take<uint64_t>(n); pa = c.take<uint32_t>(n); pb = c.take<uint32_t>(n); sk = c.take<uint32_t>(n);
    }));
    iota_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(pa, n);
    size_t temp = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp, (const uint64_t*)kin, kout, (const uint32_t*)pa, pb, (int64_t)n, 0, 64, s));
    RC(d_cub.reserve(ctx, temp));
    uint32_t* cur = pa;
    uint32_t* nxt = pb;
    for (int w = 3; w >= 0; --w) { // least significant word first
        key_word_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(d_hashes, cur, n, (uint32_t)w, kin);
        CU(cub::DeviceRadixSort::SortPairs(d_cub.ptr, temp, (const uint64_t*)kin, kout, (const uint32_t*)cur, nxt, (int64_t)n, 0, 64, s));
        uint32_t* tsw = cur; cur = nxt; nxt = tsw;
        stats.launches += 2;
    }
    if (d_seg) {
        gather_u32_kernel<<<grid1d(device, n, 256), 256, 0, s>>>(d_seg, cur, n, sk);
        size_t temp2 = 0;
        CU(cub::DeviceRadixSort::SortPairs(nullptr, temp2, (const uint32_t*)sk, (uint32_t*)kout, (const uint32_t*)cur, nxt, (int64_t)n, 0, 32, s));
        RC(d_cub.reserve(ctx, temp2));
        // d_cub may have moved: temp storage is only used inside each call, so this is safe
        CU(cub::DeviceRadixSort::SortPairs(d_cub.ptr, temp2, (const uint32_t*)sk, (uint32_t*)kout, (const uint32_t*)cur, nxt, (int64_t)n, 0, 32, s));
        uint32_t* tsw = cur; cur = nxt; nxt = tsw;
        stats.launches += 2;
    }
    CU(cudaMemcpyAsync(d_perm_out, cur, 4ull * n, cudaMemcpyDeviceToDevice, s));
    return PHANT_GPU_OK;
}

namespace {
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
    static const uint8_t EMPTY[32] = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                      0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};
    if (n == 0) {
        if (subtree_mask) { *subtree_mask = 0; memset(out_root, 0, 16 * 32); }
        else memcpy(out_root, EMPTY, 32);
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
    uint32_t *seg_cnt, *seg_off, *acc_of_slot, *kept, *perm, *slot_sorted;
    uint8_t* keep;
    RC(carve(ctx, ctx->st_seg, [&](Carve& c) {
        seg_cnt = c.take<uint32_t>(n + 2); seg_off = c.take<uint32_t>(n + 2); acc_of_slot = c.take<uint32_t>(n_slots + 1);
        kept = c.take<uint32_t>(n_slots + 1);        // compacted -> slot
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
        RC(ctx->d_b3.reserve(ctx, 64));
        size_t temp = 0;
        CU(cub::DeviceSelect::Flagged(nullptr, temp, (const uint32_t*)perm, (const uint8_t*)keep, kept, (uint32_t*)ctx->d_b3.ptr, (int64_t)n_slots, s));
        RC(ctx->d_cub.reserve(ctx, temp));
        CU(cub::DeviceSelect::Flagged(ctx->d_cub.ptr, temp, (const uint32_t*)perm, (const uint8_t*)keep, kept, (uint32_t*)ctx->d_b3.ptr, (int64_t)n_slots, s));
        CU(cudaMemcpyAsync(&m, ctx->d_b3.ptr, 4, cudaMemcpyDeviceToHost, s));
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
        RC(ctx->sort_by_segment_and_hash(ch, cacc, m, perm, ctx->st_sort));
        gather_u32_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(kept, perm, m, slot_sorted);
        gather_u32_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(cacc, perm, m, acc_sorted);
        count_per_account_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(acc_sorted, m, seg_cnt);
        storage_value_size_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(sval, slot_sorted, m, fvs);
        ctx->stats.launches += 4;
        RC(scan_sizes(ctx, fvs, fvo, m));
        storage_fill_kernel<<<grid1d(dev, m + 1, 256), 256, 0, s>>>(h_slot, sval, slot_sorted, m, fvo, fk, fko, fv);
        ctx->stats.launches++;
        size_t temp = 0;
        CU(cub::DeviceScan::ExclusiveSum(nullptr, temp, (const uint32_t*)seg_cnt, seg_off, (int64_t)(n + 1), s));
        RC(ctx->d_cub.reserve(ctx, temp));
        CU(cub::DeviceScan::ExclusiveSum(ctx->d_cub.ptr, temp, (const uint32_t*)seg_cnt, seg_off, (int64_t)(n + 1), s));
        RC(ctx->build_forest(fk, fko, fv, fvo, m, seg_off, (uint32_t)n, acc_sorted, sroots, /*32-byte keys, values <= 33 B*/ 96));
    } else {
        CU(cudaMemsetAsync(seg_off, 0, 4ull * (n + 2), s));
        RC(ctx->build_forest(nullptr, seg_off, nullptr, nullptr, 0, seg_off, (uint32_t)n, nullptr, sroots)); // every storage trie empty
    }

    // ---- account trie ----
    uint32_t *acc_perm, *ako;
    uint8_t *ak, *av;
    uint64_t *avs, *avo;
    RC(carve(ctx, ctx->st_acc, [&](Carve& c) {
        acc_perm = c.take<uint32_t>(n); ak = c.take<uint8_t>(32ull * n); ako = c.take<uint32_t>(n + 1);
        avs = c.take<uint64_t>(n + 1); avo = c.take<uint64_t>(n + 1); av = c.take<uint8_t>(112ull * n);
    }));
    RC(ctx->sort_by_segment_and_hash(h_addr, nullptr, (uint32_t)n, acc_perm, ctx->st_sort));
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
        CU(cudaMemcpyAsync(seg, ctx->d_first.ptr, sizeof seg, cudaMemcpyDeviceToHost, s));
        RC(ctx->build_forest(ak, ako, av, avo, (uint32_t)n, (const uint32_t*)ctx->d_first.ptr, 16, nullptr, (uint8_t*)ctx->d_roots.ptr,
                             160, /*the root branch consumed nibble 0*/ 1));
        CU(cudaMemcpyAsync(out_root, ctx->d_roots.ptr, 16 * 32, cudaMemcpyDeviceToHost, s));
        ctx->stats.d2h_bytes += 16 * 32 + sizeof seg;
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
    RC(ctx->build_forest(ak, ako, av, avo, (uint32_t)n, (const uint32_t*)ctx->d_first.ptr, 1, nullptr, (uint8_t*)ctx->d_roots.ptr,
                         /*32-byte keys, account RLP <= 110 B*/ 160));
    CU(cudaMemcpyAsync(out_root, ctx->d_roots.ptr, 32, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += 32;
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
    DevBuf store, work;
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
// branch node over 16 resident child hashes: f9 0211 | 16 x (a0 hash) | 80  (mpt.zig:218-247), 532 bytes, written to the arena
// parents: list of parent positions (nullable = identity).  16 threads per parent, 33 bytes each.
__global__ void ctrie_branch_encode_kernel(const uint8_t* __restrict__ child_level, const uint32_t* __restrict__ parents, uint64_t cnt,
                                           uint8_t* __restrict__ arena)
{
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t v = threadIdx.x & 15;
    for (uint64_t u = gid >> 4; u < cnt; u += ((uint64_t)gridDim.x * blockDim.x) >> 4) {
        const uint64_t p = parents ? parents[u] : u;
        uint8_t* out = arena + 532 * u;
        if (v == 0) { out[0] = 0xf9; out[1] = 0x02; out[2] = 0x11; out[531] = 0x80; }
        const uint4* h = reinterpret_cast<const uint4*>(child_level + 32 * (16 * p + v));
        const uint4 a = h[0], b = h[1];
        uint8_t* q = out + 3 + 33 * v;
        q[0] = 0xa0;
        const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            q[1 + 4 * i] = (uint8_t)w[i]; q[2 + 4 * i] = (uint8_t)(w[i] >> 8);
            q[3 + 4 * i] = (uint8_t)(w[i] >> 16); q[4 + 4 * i] = (uint8_t)(w[i] >> 24);
        }
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
__global__ void shift4_kernel(const uint32_t* __restrict__ in, uint64_t n, uint32_t* __restrict__ out)
{
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) out[k] = in[k] >> 4;
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

int ctrie_hash_level(phant_gpu_trie* t, uint32_t l, const uint32_t* d_parents, uint64_t cnt)
{
    // re-hash `cnt` branch nodes of level l (positions d_parents) from level l+1
    phant_gpu_ctx* ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    const uint64_t batch = 1ull << 20; // bound the scratch arena (532 B per node)
    for (uint64_t b0 = 0; b0 < cnt; b0 += batch) {
        const uint64_t c = cnt - b0 < batch ? cnt - b0 : batch;
        uint8_t *arena, *dg; // dg: digests are stored as 128-bit words
        uint64_t* offs;
        RC(carve(ctx, t->work, [&](Carve& w) { arena = w.take<uint8_t>(532 * c + 64); offs = w.take<uint64_t>(c + 2); dg = w.take<uint8_t>(32 * c); }));
        const uint32_t* par = d_parents + b0;
        fixed_offsets_kernel<<<grid1d(ctx->device, c, 256), 256, 0, s>>>(offs, c, 532);
        ctrie_branch_encode_kernel<<<grid1d(ctx->device, c, 128, 16), 128, 0, s>>>(t->level[l + 1], par, c, arena);
        ctx->stats.launches += 2;
        const uint32_t saved = ctx->flags;
        ctx->flags |= PHANT_GPU_FLAG_NO_BINNING; // all 532-byte messages: nothing to regroup
        const int rc = ctx->hash_csr(arena, offs, c, 532 * c, dg);
        ctx->flags = saved;
        RC(rc);
        ctrie_scatter_kernel<<<grid1d(ctx->device, c, 256), 256, 0, s>>>(dg, par, c, t->level[l]);
        ctx->stats.launches++;
    }
    CU(cudaGetLastError());
    return PHANT_GPU_OK;
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

constexpr uint8_t EMPTY_ROOT_H[32] = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                      0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};

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

int st_scan_u32(phant_gpu_ctx* ctx, const uint32_t* in, uint32_t* out, uint64_t cnt)
{
    size_t temp = 0;
    CU(cub::DeviceScan::ExclusiveSum(nullptr, temp, in, out, (int64_t)cnt, ctx->stream));
    RC(ctx->d_cub.reserve(ctx, temp));
    CU(cub::DeviceScan::ExclusiveSum(ctx->d_cub.ptr, temp, in, out, (int64_t)cnt, ctx->stream));
    return 0;
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
    RC(st_scan_u32(ctx, keep, K, n + 1));
    RC(st_scan_u32(ctx, ins_at, I, n + 2));
    if (m) RC(st_scan_u32(ctx, ins_flag, ins_index, m));
    if (n) rs_merge_table_kernel<Row><<<grid1d(dev, n, 256), 256, 0, s>>>((const Row*)table[cur].ptr, n, del_flag, K, I, (Row*)table[nxt].ptr);
    if (m) rs_merge_dirty_kernel<Row><<<grid1d(dev, m, 256), 256, 0, s>>>(dirty, kind, lb, ins_index, m, K, (Row*)table[nxt].ptr);
    ctx->stats.launches += 6;
    cur = nxt;
    return PHANT_GPU_OK;
}

// (re)build the listed buckets (d_list == nullptr: all 16^L of them) and the dense levels above them; root -> sp->root
int st_rebuild(phant_gpu_trie* t, const uint32_t* d_list, uint32_t nb, bool all)
{
    phant_gpu_ctx* ctx = t->ctx;
    SparseTrie* sp = t->sp;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    const uint32_t L = sp->L, n = (uint32_t)sp->n;
    KRow* table = (KRow*)sp->rows[sp->cur].ptr;
    uint8_t* top = (uint8_t*)sp->top.ptr;
    uint8_t* pres = (uint8_t*)sp->present.ptr;
    if (n == 0) { memcpy(sp->root, EMPTY_ROOT_H, 32); return PHANT_GPU_OK; }
    PhaseTrace tr(s);
    // per bucket: table range, size, root; per dense node: parent lists
    uint32_t *lo, *cnt, *seg_off, *par, *flag, *pos, *ping[2];
    uint8_t* roots;
    RC(carve(ctx, sp->buckets, [&](Carve& c) {
        lo = c.take<uint32_t>(nb + 2); cnt = c.take<uint32_t>(nb + 2); seg_off = c.take<uint32_t>(nb + 2); roots = c.take<uint8_t>(32ull * nb);
        par = c.take<uint32_t>(nb + 2); flag = c.take<uint32_t>(nb + 2); pos = c.take<uint32_t>(nb + 2); // parents, first-of-parent flags, positions
        ping[0] = c.take<uint32_t>(nb + 2); ping[1] = c.take<uint32_t>(nb + 2);                           // two parent lists
    }));
    st_bucket_range_kernel<<<grid1d(dev, nb, 128), 128, 0, s>>>(table, n, L, d_list, nb, lo, cnt);
    CU(cudaMemsetAsync(cnt + nb, 0, 4, s));
    RC(st_scan_u32(ctx, cnt, seg_off, nb + 1));
    uint32_t mk = 0;
    CU(cudaMemcpyAsync(&mk, seg_off + nb, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    if (mk) {
        uint8_t *gkeys, *gcache, *gcache_out;
        uint32_t *gkoff, *seg_of_key;
        uint64_t *gsize, *gvoff;
        SRec* grec;
        RC(carve(ctx, sp->gather, [&](Carve& g) {
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
        RC(sp->gvals.reserve(ctx, vbytes + 64));
        st_gather_vals_kernel<<<grid1d(dev, mk, 256, 32), 256, 0, s>>>((const uint8_t*)sp->arena.ptr, grec, gvoff, mk, (uint8_t*)sp->gvals.ptr);
        ctx->stats.launches += 3;
        tr.mark("  bucket ranges + gathers");
        RC(ctx->build_forest(gkeys, gkoff, (const uint8_t*)sp->gvals.ptr, gvoff, mk, seg_off, nb, seg_of_key, roots, -1, L, gcache, gcache_out));
        tr.mark("  build_forest");
        st_scatter_cache_kernel<<<grid1d(dev, nb, 256, 32), 256, 0, s>>>(lo, seg_off, nb, gcache_out, table);
        ctx->stats.launches++;
    }
    if (L == 0) { // one bucket: its root is the trie's root
        CU(cudaMemcpyAsync(sp->root, roots, 32, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        return PHANT_GPU_OK;
    }
    st_scatter_roots_kernel<<<grid1d(dev, nb, 256), 256, 0, s>>>(roots, d_list, cnt, nb, top + 32 * level_base(L), pres + level_base(L));
    ctx->stats.launches++;
    // dense levels bottom-up: parents of the dirty children
    static bool attr[64] = {false};
    bool& opted = attr[(dev >= 0 && dev < 64) ? dev : 0];
    if (!opted) { CU(cudaFuncSetAttribute(st_top_branch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FR_SMEM)); opted = true; }
    RC(ctx->d_b3.reserve(ctx, 64));
    uint32_t* viol = (uint32_t*)ctx->d_b3.ptr + 12;
    CU(cudaMemsetAsync(viol, 0, 4, s));
    const uint32_t* child = d_list;
    uint32_t cbound = nb;                       // upper bound of the children count; the exact count stays on the device
    uint32_t* cnt_dev = (uint32_t*)ctx->d_b3.ptr + 13;
    CU(cudaMemcpyAsync(cnt_dev, &nb, 4, cudaMemcpyHostToDevice, s));
    const unsigned fr_cap = (unsigned)keccak_num_sms(dev) * 3;
    for (int d = (int)L - 1; d >= 0; --d) {
        const uint32_t* plist = nullptr;
        uint32_t pbound = 1u << (4 * d);
        const uint32_t* pcount_dev = nullptr;
        if (!all) { // distinct parents of the (sorted) dirty children
            uint32_t* uniq = ping[d & 1];
            st_parent_flag_kernel<<<grid1d(dev, cbound + 1, 256), 256, 0, s>>>(child, cnt_dev, cbound, par, flag);
            RC(st_scan_u32(ctx, flag, pos, cbound + 1));
            st_compact_kernel<<<grid1d(dev, cbound, 256), 256, 0, s>>>(par, flag, pos, cbound, uniq);
            CU(cudaMemcpyAsync(cnt_dev, pos + cbound, 4, cudaMemcpyDeviceToDevice, s)); // the parents are the next level's children
            if (cbound < pbound) pbound = cbound;
            plist = uniq;
            child = uniq;
            cbound = pbound;
            pcount_dev = cnt_dev;
            ctx->stats.launches += 3;
        }
        const unsigned g = (pbound + FR_WARPS * 32 - 1) / (FR_WARPS * 32);
        st_top_branch_kernel<<<g < fr_cap ? g : fr_cap, FR_WARPS * 32, FR_SMEM, s>>>(top + 32 * level_base(d + 1), pres + level_base(d + 1), plist, nullptr, nullptr,
                                                                               pbound, pcount_dev,
                                                                               top + 32 * level_base(d), pres + level_base(d), viol);
        ctx->stats.launches++;
    }
    CU(cudaGetLastError());
    tr.mark("  dense levels");
    uint32_t v = 0;
    CU(cudaMemcpyAsync(sp->root, top, 32, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&v, viol, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return v ? 1 : PHANT_GPU_OK; // 1 = the dense-top premise does not hold at this L
}

int st_set_L_and_rebuild_all(phant_gpu_trie* t, uint32_t L)
{
    phant_gpu_ctx* ctx = t->ctx;
    SparseTrie* sp = t->sp;
    for (;;) {
        sp->L = L;
        const uint64_t nodes = level_base(L + 1);
        RC(sp->top.reserve(ctx, 32 * nodes + 64));
        RC(sp->present.reserve(ctx, nodes + 64));
        CU(cudaMemsetAsync(sp->present.ptr, 0, nodes, ctx->stream));
        sp->rebuilds++;
        const int rc = st_rebuild(t, nullptr, 1u << (4 * L), true);
        if (rc != 1) return rc;
        if (L == 0) return PHANT_GPU_E_CUDA; // cannot happen: L = 0 has no dense level
        --L; // some top node has a single child: fewer dense levels
    }
}

// Everything an update of m keys with vb value bytes works in (sp->dirty), laid out in one place so that a caller can reserve
// it before its first write: the staging area the caller fills on the device (the dirty keys as given, the values, their
// m+1 offsets), the sorted dirty rows with their classification, and the merge scratch of the n-row table.
struct StrieDirty {
    uint8_t* keys; uint8_t* vals; uint32_t* val_off;
    uint32_t* perm; KRow* rows; uint8_t* del; uint8_t* kind;
    uint32_t *lb, *ins_flag, *ins_index, *bucket;
    uint32_t *del_flag, *ins_at, *keep, *K, *I;
};
int strie_dirty_area(phant_gpu_trie* t, uint32_t m, uint64_t vb, StrieDirty* a)
{
    const uint64_t n = t->sp->n;
    RC(carve(t->ctx, t->sp->dirty, [&](Carve& c) {
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
int strie_compact_arena(phant_gpu_trie* t)
{
    phant_gpu_ctx* ctx = t->ctx;
    SparseTrie* sp = t->sp;
    cudaStream_t s = ctx->stream;
    const uint32_t n = (uint32_t)sp->n;
    KRow* rows = (KRow*)sp->rows[sp->cur].ptr;
    uint64_t *len, *off;
    RC(carve(ctx, sp->gather, [&](Carve& c) { len = c.take<uint64_t>(n + 1); off = c.take<uint64_t>(n + 1); }));
    st_rec_len_kernel<<<grid1d(ctx->device, n, 256), 256, 0, s>>>(rows, n, len);
    RC(scan_sizes(ctx, len, off, n));
    uint64_t live = 0;
    CU(cudaMemcpyAsync(&live, off + n, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    DevBuf fresh;
    RC(fresh.reserve(ctx, 2ull * sp->compact_row * n + (1 << 20)));
    st_gather_vals_kernel<<<grid1d(ctx->device, n, 256, 32), 256, 0, s>>>((const uint8_t*)sp->arena.ptr, rows, off, n, (uint8_t*)fresh.ptr);
    st_rebase_recs_kernel<<<grid1d(ctx->device, n, 256), 256, 0, s>>>(rows, n, off);
    ctx->stats.launches += 4;
    CU(cudaStreamSynchronize(s));
    sp->arena.release();
    sp->arena = fresh;
    sp->arena_used = live;
    return PHANT_GPU_OK;
}

// The update itself, from the staged dirty area (strie_dirty_area), which the caller filled on the device.
int strie_apply(phant_gpu_trie* t, uint32_t m, uint64_t vb, uint8_t out_root[32])
{
    phant_gpu_ctx* ctx = t->ctx;
    SparseTrie* sp = t->sp;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    if (m == 0) { memcpy(out_root, sp->root, 32); return PHANT_GPU_OK; }
    const uint32_t n = (uint32_t)sp->n;
    StrieDirty a;
    RC(strie_dirty_area(t, m, vb, &a));
    PhaseTrace tr(s);
    RC(ctx->sort_by_segment_and_hash(a.keys, nullptr, m, a.perm, sp->sort));
    tr.mark("sort dirty keys");
    // ---- dirty rows, classified against the table ----
    CU(cudaMemsetAsync(a.del_flag, 0, 4ull * (n + 3) * 2, s));
    RC(ctx->d_b3.reserve(ctx, 64));
    uint32_t* counters = (uint32_t*)ctx->d_b3.ptr;
    CU(cudaMemsetAsync(counters, 0, 64, s));
    st_dirty_rows_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(a.keys, a.val_off, a.perm, m, sp->arena_used, a.rows, a.del, counters);
    KRow* table = (KRow*)sp->rows[sp->cur].ptr;
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
    if (sp->arena_used + app_bytes + 64 > sp->arena.cap) {
        DevBuf bigger;
        RC(bigger.reserve(ctx, (sp->arena_used + app_bytes) * 2 + (1 << 20)));
        if (sp->arena_used) CU(cudaMemcpyAsync(bigger.ptr, sp->arena.ptr, sp->arena_used, cudaMemcpyDeviceToDevice, s));
        CU(cudaStreamSynchronize(s));
        sp->arena.release();
        sp->arena = bigger;
    }
    if (app_bytes) CU(cudaMemcpyAsync((uint8_t*)sp->arena.ptr + sp->arena_used, a.vals + v0, app_bytes, cudaMemcpyDeviceToDevice, s));
    sp->arena_used += app_bytes;
    // ---- replaced rows in place (a new value: no cached leaf reference), then the merge (skipped for pure value updates) ----
    rs_replace_kernel<KRow><<<grid1d(dev, m, 256), 256, 0, s>>>(a.rows, a.kind, a.lb, m, table);
    ctx->stats.launches++;
    const uint32_t new_n = n - n_del + n_ins;
    if (n_ins || n_del) {
        RC(sp->rows[1 - sp->cur].reserve(ctx, sizeof(KRow) * new_n + 64));
        RC(rs_merge<KRow>(ctx, sp->rows, sp->cur, n, a.rows, m, a.kind, a.lb, a.ins_flag, a.del_flag, a.ins_at, a.keep, a.K, a.I, a.ins_index));
        sp->n = new_n;
    }
    tr.mark("merge");
    sp->updates++;
    if (new_n == 0) {
        sp->L = 0;
        memcpy(sp->root, EMPTY_ROOT_H, 32);
        memcpy(out_root, sp->root, 32);
        return PHANT_GPU_OK;
    }
    // ---- which part of the trie to re-hash ----
    const uint32_t Lt = st_target_L(new_n);
    int rc;
    if (Lt > sp->L || Lt + 1 < sp->L || n == 0) {
        rc = st_set_L_and_rebuild_all(t, Lt);      // the table grew / shrank past a bucket-size bound: new dense depth
    } else {
        uint32_t* first = a.ins_flag;               // (classification scratch is free again)
        uint32_t* fpos = a.ins_index;
        uint32_t* list = a.lb;
        st_bucket_flag_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(a.rows, m, sp->L, a.bucket, first);
        CU(cudaMemsetAsync(first + m, 0, 4, s));
        RC(st_scan_u32(ctx, first, fpos, m + 1));
        st_compact_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(a.bucket, first, fpos, m, list);
        uint32_t nb = 0;
        CU(cudaMemcpyAsync(&nb, fpos + m, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches += 3;
        rc = st_rebuild(t, list, nb, false);
        if (rc == 1) rc = st_set_L_and_rebuild_all(t, sp->L - 1); // a dense node lost all but one child: fewer dense levels
    }
    tr.mark("rebuild (buckets + top)");
    if (rc) return rc;
    if (sp->compact && sp->arena_used > 2ull * sp->compact_row * sp->n + (1 << 20)) RC(strie_compact_arena(t)); // over half of it is dead
    memcpy(out_root, sp->root, 32);
    ctx->stats.d2h_bytes += 36;
    return PHANT_GPU_OK;
}

int strie_update(phant_gpu_trie* t, const uint8_t* keys32, const uint8_t* vals, const uint32_t* val_off, uint64_t m64, uint8_t out_root[32])
{
    phant_gpu_ctx* ctx = t->ctx;
    SparseTrie* sp = t->sp;
    cudaStream_t s = ctx->stream;
    if (ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) return PHANT_GPU_E_INVALID; // host tables (it is the StateDB flattening, as S)
    if (m64 == 0) { memcpy(out_root, sp->root, 32); return PHANT_GPU_OK; }
    if (!keys32 || !val_off || m64 >= (1ull << 28) || sp->n + m64 >= (1ull << 30)) return PHANT_GPU_E_INVALID;
    const uint32_t m = (uint32_t)m64;
    for (uint32_t i = 0; i < m; ++i)
        if (val_off[i + 1] < val_off[i]) return PHANT_GPU_E_INVALID;
    const uint64_t vb = val_off[m];
    if (vb && !vals) return PHANT_GPU_E_INVALID;
    StrieDirty area;
    RC(strie_dirty_area(t, m, vb, &area));
    PhaseTrace tr(s);
    CU(cudaMemcpyAsync(area.keys, keys32, 32ull * m, cudaMemcpyHostToDevice, s));
    if (vb) CU(cudaMemcpyAsync(area.vals, vals, vb, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(area.val_off, val_off, 4ull * (m + 1), cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += 32ull * m + vb + 4ull * (m + 1);
    tr.mark("stage dirty (H2D)");
    return strie_apply(t, m, vb, out_root);
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
    // all branch levels bottom-up; explicit parent lists keep the batches simple
    for (int l = (int)desc->depth - 1; l >= 0; --l) {
        uint64_t n_l = 1;
        for (int k = 0; k < l; ++k) n_l *= 16;
        DevBuf ids;
        if (int rc = ids.reserve(ctx, 4 * n_l + 16)) { t->store.release(); delete t; return rc; }
        iota_kernel<<<grid1d(ctx->device, n_l, 256), 256, 0, ctx->stream>>>((uint32_t*)ids.ptr, (uint32_t)n_l);
        int rc = ctrie_hash_level(t, (uint32_t)l, (const uint32_t*)ids.ptr, n_l);
        cudaStreamSynchronize(ctx->stream);
        ids.release();
        if (rc) { t->store.release(); t->work.release(); delete t; return rc; }
    }
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
    if (t->kind == 1) return strie_update(t, keys32, leaf_vals, val_off, n_dirty, out_root);
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
    if (!(ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS) && max_val <= FR_SLOT - 48) {
        // ---- fused frontier path: one launch for the leaves, then per level shift/pad + unique + one hash launch; the only
        // host synchronisation is the final read of the root ----
        static bool attr[64] = {false}; // function attributes are per device (as launch_staged in keccak_kernels.cu)
        bool& opted = attr[(ctx->device >= 0 && ctx->device < 64) ? ctx->device : 0];
        if (!opted) {
            CU(cudaFuncSetAttribute(frontier_branch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FR_SMEM));
            CU(cudaFuncSetAttribute(frontier_leaf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FR_SMEM));
            opted = true;
        }
        uint32_t *pos, *cur, *tmp, *uniq;
        RC(carve(ctx, ctx->d_b0, [&](Carve& c) {
            pos = c.take<uint32_t>(n_dirty); cur = c.take<uint32_t>(n_dirty); tmp = c.take<uint32_t>(n_dirty); uniq = c.take<uint32_t>(n_dirty);
        }));
        RC(ctx->d_b3.reserve(ctx, 64));
        uint32_t* counts = (uint32_t*)ctx->d_b3.ptr; // counts[0] = valid entries of `cur`; counts[8] = "refused" flag
        uint32_t* refuse = counts + 8;
        const unsigned fr_grid = (unsigned)((n_dirty + FR_WARPS * 32 - 1) / (FR_WARPS * 32));
        const unsigned fr_cap = (unsigned)keccak_num_sms(ctx->device) * 3;
        // positions first, sorted, checked for collisions; only then is anything written to the resident levels
        ctrie_leaf_pos_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_keys, n_dirty, L, pos);
        size_t temp = 0;
        CU(cub::DeviceRadixSort::SortKeys(nullptr, temp, (const uint32_t*)pos, cur, (int64_t)n_dirty, 0, 4 * (int)L, s));
        RC(ctx->d_cub.reserve(ctx, temp));
        CU(cub::DeviceRadixSort::SortKeys(ctx->d_cub.ptr, temp, (const uint32_t*)pos, cur, (int64_t)n_dirty, 0, 4 * (int)L, s));
        const uint32_t init[16] = {(uint32_t)n_dirty, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        CU(cudaMemcpyAsync(counts, init, sizeof init, cudaMemcpyHostToDevice, s));
        ctrie_dup_check_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(cur, n_dirty, refuse);
        frontier_leaf_kernel<<<fr_grid < fr_cap ? fr_grid : fr_cap, FR_WARPS * 32, FR_SMEM, s>>>(d_keys, d_vals, d_voff, (uint32_t)n_dirty, L, t->level[L], pos, refuse);
        ctx->stats.launches += 4;
        uint64_t bound = n_dirty;
        for (int l = (int)L - 1; l >= 0; --l) {
            shift4_pad_kernel<<<grid1d(ctx->device, bound, 256), 256, 0, s>>>(cur, counts, (uint32_t)bound, tmp);
            size_t t2 = 0;
            CU(cub::DeviceSelect::Unique(nullptr, t2, (const uint32_t*)tmp, uniq, counts, (int64_t)bound, s));
            RC(ctx->d_cub.reserve(ctx, t2));
            CU(cub::DeviceSelect::Unique(ctx->d_cub.ptr, t2, (const uint32_t*)tmp, uniq, counts, (int64_t)bound, s));
            uint64_t level_nodes = 1;
            for (int q = 0; q < l; ++q) level_nodes *= 16;
            if (bound > level_nodes) bound = level_nodes; // a level cannot have more dirty nodes than nodes
            const unsigned g = (unsigned)((bound + FR_WARPS * 32 - 1) / (FR_WARPS * 32));
            frontier_branch_kernel<<<g < fr_cap ? g : fr_cap, FR_WARPS * 32, FR_SMEM, s>>>(t->level[l + 1], uniq, counts, (uint32_t)bound, t->level[l], refuse);
            ctx->stats.launches += 3;
            uint32_t* x = cur; cur = uniq; uniq = x;
        }
        CU(cudaGetLastError());
        uint32_t refused = 0;
        CU(cudaMemcpyAsync(out_root, t->level[0], 32, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(&refused, refuse, 4, cudaMemcpyDeviceToHost, s));
        ctx->stats.d2h_bytes += 36;
        CU(cudaStreamSynchronize(s));
        return refused ? PHANT_GPU_E_INVALID : PHANT_GPU_OK; // refused: the trie is unchanged, out_root = its current root
    }
    // ---- general path (device pointers, or leaf values too large for a staging slot):
    // dirty leaves: encode, hash (batched Keccak), scatter into the leaf level ----
    uint32_t *pos, *pa, *pb, *pc;
    uint64_t *sizes, *offs;
    uint8_t* dg;
    RC(carve(ctx, ctx->d_b0, [&](Carve& c) {
        pos = c.take<uint32_t>(n_dirty); pa = c.take<uint32_t>(n_dirty); pb = c.take<uint32_t>(n_dirty); pc = c.take<uint32_t>(n_dirty);
        sizes = c.take<uint64_t>(n_dirty + 2); offs = c.take<uint64_t>(n_dirty + 2); dg = c.take<uint8_t>(32 * n_dirty);
    }));
    ctrie_leaf_pos_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_keys, n_dirty, L, pos);
    {   // distinct leaf positions, checked before anything is written to the resident levels
        size_t temp0 = 0;
        CU(cub::DeviceRadixSort::SortKeys(nullptr, temp0, (const uint32_t*)pos, pa, (int64_t)n_dirty, 0, 4 * (int)L, s));
        RC(ctx->d_cub.reserve(ctx, temp0));
        CU(cub::DeviceRadixSort::SortKeys(ctx->d_cub.ptr, temp0, (const uint32_t*)pos, pa, (int64_t)n_dirty, 0, 4 * (int)L, s));
        RC(ctx->d_b3.reserve(ctx, 64));
        CU(cudaMemsetAsync(ctx->d_b3.ptr, 0, 64, s));
        ctrie_dup_check_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(pa, n_dirty, (uint32_t*)ctx->d_b3.ptr);
        uint32_t refused = 0;
        CU(cudaMemcpyAsync(&refused, ctx->d_b3.ptr, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches += 2;
        if (refused) return PHANT_GPU_E_INVALID;
    }
    ctrie_leaf_size_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_vals, d_voff, n_dirty, L, sizes);
    RC(scan_sizes(ctx, sizes, offs, n_dirty));
    uint64_t total = 0;
    CU(cudaMemcpyAsync(&total, offs + n_dirty, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    RC(ctx->d_b1.reserve(ctx, total + 64));
    ctrie_leaf_encode_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(d_keys, d_vals, d_voff, n_dirty, L, offs, (uint8_t*)ctx->d_b1.ptr);
    ctx->stats.launches += 3;
    RC(ctx->hash_csr((const uint8_t*)ctx->d_b1.ptr, offs, n_dirty, total, dg));
    ctrie_scatter_kernel<<<grid1d(ctx->device, n_dirty, 256), 256, 0, s>>>(dg, pos, n_dirty, t->level[L]);
    ctx->stats.launches++;
    // ---- frontier: unique parents level by level (`pa` = the sorted positions, then shift + unique) ----
    uint64_t cnt = n_dirty;
    uint32_t* cur = pa;
    uint32_t* tmp = pb;
    uint32_t* uniq = pc;
    for (int l = (int)L - 1; l >= 0; --l) {
        shift4_kernel<<<grid1d(ctx->device, cnt, 256), 256, 0, s>>>(cur, cnt, tmp);
        size_t t2 = 0;
        CU(cub::DeviceSelect::Unique(nullptr, t2, (const uint32_t*)tmp, uniq, (uint32_t*)ctx->d_b3.ptr, (int64_t)cnt, s));
        RC(ctx->d_cub.reserve(ctx, t2));
        CU(cub::DeviceSelect::Unique(ctx->d_cub.ptr, t2, (const uint32_t*)tmp, uniq, (uint32_t*)ctx->d_b3.ptr, (int64_t)cnt, s));
        uint32_t nu = 0;
        CU(cudaMemcpyAsync(&nu, ctx->d_b3.ptr, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ctx->stats.launches += 2;
        cnt = nu;
        RC(ctrie_hash_level(t, (uint32_t)l, uniq, cnt));
        uint32_t* x = cur; cur = uniq; uniq = x; // the unique parents are the next level's (sorted) children
    }
    CU(cudaMemcpyAsync(out_root, t->level[0], 32, cudaMemcpyDeviceToHost, s));
    ctx->stats.d2h_bytes += 32;
    CU(cudaStreamSynchronize(s));
    return PHANT_GPU_OK;
}

extern "C" void phant_gpu_trie_close(phant_gpu_trie* t)
{
    if (!t) return;
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    t->store.release();
    t->work.release();
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
// P's account-body decoder, for the old account of an undo record.  Its header opens an anonymous namespace inside `phant`;
// wrapped in a namespace of its own so that it does not meet this file's anonymous namespace through `using namespace phant`.
namespace rs_body {
#include "state_read.cuh"
}
using rs_body::phant::AccountBody;
using rs_body::phant::decode_account_body;
namespace {

// ---- undo records (phant_gpu_resident_state_set_journal): the inverse of an apply, captured from the pre-merge tables ----
// listed slots [lo, hi) of listed account i (sorted by account)
__device__ __forceinline__ void listed_slots(const uint32_t* sacc, uint32_t ms, uint32_t i, uint32_t& lo, uint32_t& hi)
{
    uint32_t a = 0, b = ms;
    while (a < b) { const uint32_t mid = (a + b) >> 1; if (sacc[mid] < i) a = mid + 1; else b = mid; }
    uint32_t c = a, d = ms;
    while (c < d) { const uint32_t mid = (c + d) >> 1; if (sacc[mid] < i + 1) c = mid + 1; else d = mid; }
    lo = a;
    hi = c;
}
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

} // namespace

struct phant_gpu_resident_state {
    phant_gpu_ctx* ctx;
    phant_gpu_trie acct;   // kind 1: account key -> rlp([nonce, balance, storageRoot, codeHash])
    SparseTrie acct_sp;
    DevBuf S[2], A[2], pool[2]; // slot table, account rows, dense-top pool (32-byte references, then presence bytes)
    int sc = 0, ac = 0, pc = 0;
    uint32_t nS = 0, nA = 0;
    uint64_t pool_nodes = 0;
    DevBuf in, dirty, work, forest, sort; // scratch
    bool writing = false; // the current apply has started to change resident data
    bool failed = false;  // an apply failed after its first write: the tables may disagree, every later call is refused
    // undo journal: one record per successful apply, newest last; a record is a diff on the device (the staging layout) that
    // takes the state back to `root`
    struct Record { DevBuf buf; uint32_t na = 0, ms = 0; uint8_t root[32]; };
    uint32_t depth = 0;
    std::deque<Record> journal;
    Record next;               // the record the current apply captures into
    std::vector<DevBuf> spare; // buffers of dropped and undone records, reused
    // witness: the exported nodes (scratch), and the result the last witness call holds until it is copied or another call comes
    DevBuf wit_out, wit_res;
    bool wit_held = false;
    uint64_t wit_n = 0, wit_bytes = 0;
    void drop_witness() { wit_res.release(); wit_held = false; }
    std::vector<DevBuf*> bufs()
    {
        std::vector<DevBuf*> v = {&S[0], &S[1], &A[0], &A[1], &pool[0], &pool[1], &in, &dirty, &work, &forest, &sort, &acct_sp.rows[0], &acct_sp.rows[1],
                &acct_sp.arena, &acct_sp.top, &acct_sp.present, &acct_sp.dirty, &acct_sp.buckets, &acct_sp.gather, &acct_sp.gvals, &acct_sp.sort,
                &wit_out, &wit_res};
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

bool is_device_ptr(const void* p)
{
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice;
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
    for (const void* q : {(const void*)d->account_keys32, (const void*)d->account_flags, (const void*)d->nonce, (const void*)d->balance32,
                          (const void*)d->code_hash32, (const void*)d->slot_account, (const void*)d->slot_keys32, (const void*)d->slot_vals32})
        if (is_device_ptr(q)) return PHANT_GPU_E_INVALID;
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
    RC(ctx->sort_by_segment_and_hash(dd.akeys, nullptr, na, f.perm_a, st->sort));
    rs_rank_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(f.perm_a, na, f.rank);
    rs_acc_dirty_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(dd.akeys, dd.aflags, f.perm_a, na, f.arows, f.adel, f.aclear, f.counters);
    ctx->stats.launches += 2;
    if (ms) {
        gather_u32_kernel<<<grid1d(dev, ms, 256), 256, 0, s>>>(f.rank, dd.sacc, ms, f.seg);
        RC(ctx->sort_by_segment_and_hash(dd.skeys, f.seg, ms, f.perm_s, st->sort));
        rs_slot_dirty_kernel<<<grid1d(dev, ms, 256), 256, 0, s>>>(dd.akeys, dd.aflags, dd.sacc, dd.skeys, dd.svals, f.seg, f.perm_s, ms, f.srows,
                                                                  f.sacc, f.sdel, f.sabs, f.counters);
        ctx->stats.launches += 2;
    }
    rs_classify_kernel<AccRow, 32><<<grid1d(dev, na, 128), 128, 0, s>>>((const AccRow*)st->A[st->ac].ptr, nA, f.arows, na, f.adel, nullptr, f.alb,
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
    RC(st_scan_u32(ctx, up_flag, up_pos, na + 1));
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
        rs_classify_kernel<SlotRow, 64><<<grid1d(dev, ms, 128), 128, 0, s>>>((const SlotRow*)st->S[st->sc].ptr, nS, f.srows, ms, f.sdel, f.sabs, slb,
                                                                            skind, del_flag, ins_at, sins, counters + 8);
        ctx->stats.launches++;
    }
    rs_clear_slots_kernel<<<grid1d(dev, na, 256, 32), 256, 0, s>>>((const SlotRow*)st->S[st->sc].ptr, nS, (const AccRow*)st->A[st->ac].ptr, f.arows,
                                                                   f.aclear, f.akind, f.alb, na, del_flag, counters);
    CU(cudaMemsetAsync(ains_cnt, 0, 4ull * na, s));
    if (ms) rs_slot_ins_count_kernel<<<grid1d(dev, ms, 256), 256, 0, s>>>(f.sacc, skind, ms, ains_cnt);
    rs_pool_bound_kernel<<<grid1d(dev, na, 128), 128, 0, s>>>((const SlotRow*)st->S[st->sc].ptr, nS, (const AccRow*)st->A[st->ac].ptr, f.arows,
                                                             f.adel, f.aclear, f.akind, f.alb, ains_cnt, na, pool_bound);
    ctx->stats.launches += ms ? 3 : 2;
    const KRow* krows = (const KRow*)st->acct_sp.rows[st->acct_sp.cur].ptr;
    const uint8_t* karena = (const uint8_t*)st->acct_sp.arena.ptr;
    if (rec) { // the undo record's size; counters[12]: an old account body that does not decode
        rs_undo_size_kernel<<<grid1d(dev, na + 1, 128), 128, 0, s>>>(f.arows, f.aclear, f.akind, f.alb, na, (const SlotRow*)st->S[st->sc].ptr, nS,
                                                                     f.sacc, ms, krows, karena, u_listed, u_nslots, counters + 12);
        RC(st_scan_u32(ctx, u_listed, u_apos, na + 1));
        RC(st_scan_u32(ctx, u_nslots, u_soff, na + 1));
        ctx->stats.launches++;
    }
    CU(cudaMemcpyAsync(hc, counters, 64, cudaMemcpyDeviceToHost, s));
    if (rec) {
        CU(cudaMemcpyAsync(hc + 13, u_apos + na, 4, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(hc + 14, u_soff + na, 4, cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    if (rec && hc[12]) { // cannot happen: the account trie's leaves are written by account_fill_kernel
        snprintf(ctx->last_error, sizeof ctx->last_error, "resident state: an account leaf of the account trie does not decode");
        return PHANT_GPU_E_CUDA;
    }
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
        RC(strie_dirty_area(&st->acct, na, 112ull * na, &area));
    }
    if (rec) { // the undo record: a diff in the staging layout, filled from the tables as they are before the merge
        RsDiff r;
        RC(carve(ctx, rec->buf, [&](Carve& c) { r.take(c, hc[13], hc[14]); }));
        rs_undo_fill_kernel<<<grid1d(dev, na, 256, 32), 256, 0, s>>>(f.arows, f.aclear, f.akind, f.alb, na, (const SlotRow*)st->S[st->sc].ptr, nS,
                                                                   f.srows, f.sacc, skind, slb, ms, krows, karena, u_apos, u_soff, r.akeys,
                                                                   r.aflags, r.nonce, r.bal, r.code, r.sacc, r.skeys, r.svals);
        ctx->stats.launches++;
        rec->na = r.na;
        rec->ms = r.ms;
    }
    st->writing = true; // from here on a failure leaves the tables half-updated

    // ---- merge both tables ----
    if (ms) {
        rs_replace_kernel<SlotRow><<<grid1d(dev, ms, 256), 256, 0, s>>>(f.srows, skind, slb, ms, (SlotRow*)st->S[st->sc].ptr);
        ctx->stats.launches++;
    }
    if (s_merge) RC(rs_merge<SlotRow>(ctx, st->S, st->sc, nS, f.srows, ms, skind, slb, sins, del_flag, ins_at, keep, Ksc, Isc, sins_index));
    if (a_merge) RC(rs_merge<AccRow>(ctx, st->A, st->ac, nA, f.arows, na, f.akind, f.alb, f.ains, f.del_flag, f.ins_at, keep, Ksc, Isc, ains_index));
    st->nS = nS_new;
    st->nA = nA_new;
    AccRow* A = (AccRow*)st->A[st->ac].ptr;
    const SlotRow* S = (const SlotRow*)st->S[st->sc].ptr;

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
        RC(st_scan_u32(ctx, first, F, ms + 1));
        rs_bucket_count_kernel<<<grid1d(dev, na + 1, 256), 256, 0, s>>>(F, na, p, cnt);
        RC(st_scan_u32(ctx, cnt, off, na + 1));
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
            RC(st_scan_u32(ctx, ecnt, seg_off, E + 1));
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
                RC(ctx->build_forest(fk, fko, fv, fvo, mk, seg_off, E, seg_of_key, roots, /*32-byte keys, values <= 33 B*/ 96, 0, nullptr, nullptr,
                                     estart));
            } else {
                RC(ctx->build_forest(nullptr, seg_off, nullptr, nullptr, 0, seg_off, E, nullptr, roots)); // every listed bucket empty
            }
            rs_scatter_roots_kernel<<<grid1d(dev, E, 256), 256, 0, s>>>(roots, e_acc, e_b, ecnt, E, p, A, top, present);
            ctx->stats.launches++;
            static bool attr[64] = {false};
            bool& opted = attr[(dev >= 0 && dev < 64) ? dev : 0];
            if (!opted) { CU(cudaFuncSetAttribute(st_top_branch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FR_SMEM)); opted = true; }
            const unsigned fr_cap = (unsigned)keccak_num_sms(dev) * 3;
            for (int dd = (int)maxL - 1; dd >= 0; --dd) { // one launch per level across all accounts
                rs_node_flag_kernel<<<grid1d(dev, E + 1, 256), 256, 0, s>>>(e_acc, e_b, E, (uint32_t)dd, p, nfirst);
                RC(st_scan_u32(ctx, nfirst, npos, E + 1));
                rs_node_list_kernel<<<grid1d(dev, E, 256), 256, 0, s>>>(e_acc, e_b, nfirst, npos, E, (uint32_t)dd, p, A, npar, nbase, nown);
                const unsigned gsz = (E + FR_WARPS * 32 - 1) / (FR_WARPS * 32);
                st_top_branch_kernel<<<gsz < fr_cap ? gsz : fr_cap, FR_WARPS * 32, FR_SMEM, s>>>(
                    top + 32 * level_base(dd + 1), present + level_base(dd + 1), npar, nbase, nown, E, npos + E, top + 32 * level_base(dd),
                    present + level_base(dd), p.viol);
                ctx->stats.launches += 4;
            }
            rs_top_root_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(na, p, A, top, present);
            ctx->stats.launches++;
        }
        // premise check of this round: any listed account whose dense top has a one-child node
        {
            size_t temp = 0;
            CU(cub::DeviceReduce::Max(nullptr, temp, p.viol, counters + 4, (int64_t)na, s));
            RC(ctx->d_cub.reserve(ctx, temp));
            CU(cub::DeviceReduce::Max(ctx->d_cub.ptr, temp, p.viol, counters + 4, (int64_t)na, s));
        }
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
    RC(strie_dirty_area(&st->acct, na, vb, &area));
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
    RC(strie_apply(&st->acct, na, vb, out_root));
    if (storage_roots32) {
        CU(cudaMemcpyAsync(storage_roots32, sroot_out, 32ull * na, cudaMemcpyDeviceToHost, s));
        ctx->stats.d2h_bytes += 32ull * na;
        CU(cudaStreamSynchronize(s));
    }
    return PHANT_GPU_OK;
}

// The pre-state witness of a diff (phant_gpu_resident_state_witness), held in st->wit_res.  The diff is staged, sorted and
// classified by the apply's kernels; the proof keys of every trie (listed keys, and the surviving neighbours of deleted ones)
// are sorted by (trie, key); the dense-top nodes on their paths are encoded from the pool; the buckets that hold a proof key
// are rebuilt as one forest whose nodes on the proof paths are exported; the exported nodes are sorted by digest and the
// duplicates dropped.  Only scratch is written.
int rs_witness(phant_gpu_resident_state* st, const phant_gpu_state_diff* d)
{
    phant_gpu_ctx* ctx = st->ctx;
    cudaStream_t s = ctx->stream;
    const int dev = ctx->device;
    st->wit_n = st->wit_bytes = 0;
    RsDiff dd;
    RC(rs_stage(st, d, dd));
    if (dd.na == 0) { st->wit_held = true; return PHANT_GPU_OK; }
    const uint32_t na = dd.na, ms = dd.ms, nS = st->nS, nA = st->nA;

    // ---- sort and classify, then list the proof-key candidates (counters[2]) ----
    const uint32_t C = 3 * na + 3 * ms; // proof-key candidates
    RsSorted f;
    uint32_t *cseg, *cperm;
    uint8_t* ckeys;
    WitTries w;
    RC(carve(ctx, st->dirty, [&](Carve& c) {
        f.take(c, na, ms, nA);
        w.ok = c.take<uint8_t>(na + 1); w.L = c.take<uint32_t>(na + 1); w.base = c.take<uint32_t>(na + 1);
        w.slo = c.take<uint32_t>(na + 1); w.shi = c.take<uint32_t>(na + 1);
        ckeys = c.take<uint8_t>(32ull * C); cseg = c.take<uint32_t>(C); cperm = c.take<uint32_t>(C);
    }));
    RC(rs_sort_classify(st, dd, f));
    const AccRow* A = (const AccRow*)st->A[st->ac].ptr;
    const SlotRow* S = (const SlotRow*)st->S[st->sc].ptr;
    const SparseTrie& sp = st->acct_sp;
    const KRow* krows = (const KRow*)sp.rows[sp.cur].ptr;
    const uint32_t n = (uint32_t)sp.n;
    wit_tries_kernel<<<grid1d(dev, na + 1, 128), 128, 0, s>>>(A, S, nS, f.arows, f.aclear, f.akind, f.alb, na, n, sp.L, w);
    wit_acc_keys_kernel<<<grid1d(dev, na, 128), 128, 0, s>>>(f.arows, f.adel, na, krows, n, ckeys, cseg, f.counters + 2);
    ctx->stats.launches += 2;
    if (ms) {
        wit_slot_keys_kernel<<<grid1d(dev, ms, 128), 128, 0, s>>>(f.srows, f.sacc, f.sdel, ms, S, nS, w, 3 * na, ckeys, cseg, f.counters + 2);
        ctx->stats.launches++;
    }
    uint32_t hc[16];
    CU(cudaMemcpyAsync(hc, f.counters, 64, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.d2h_bytes += 64;
    if (hc[0] || hc[1]) return PHANT_GPU_E_INVALID; // an account twice, or (account, slot) twice
    const uint32_t np = hc[2];
    if (np == 0) { st->wit_held = true; return PHANT_GPU_OK; } // the empty state: no node

    // ---- proof keys sorted by (trie, key); the buckets that hold one ----
    uint8_t* pkeys;
    uint32_t *ptrie, *first, *bpos;
    RC(carve(ctx, st->work, [&](Carve& c) {
        pkeys = c.take<uint8_t>(32ull * np); ptrie = c.take<uint32_t>(np); first = c.take<uint32_t>(np + 1); bpos = c.take<uint32_t>(np + 1);
    }));
    RC(ctx->sort_by_segment_and_hash(ckeys, cseg, C, cperm, st->sort)); // the NONE candidates sort last
    wit_proof_keys_kernel<<<grid1d(dev, np, 256), 256, 0, s>>>(ckeys, cseg, cperm, np, pkeys, ptrie);
    const uint8_t* pool_top = (const uint8_t*)st->pool[st->pc].ptr;
    const WitTops tp{(const uint8_t*)sp.top.ptr, (const uint8_t*)sp.present.ptr, pool_top, pool_top + 32 * st->pool_nodes};
    wit_bucket_flag_kernel<<<grid1d(dev, np + 1, 256), 256, 0, s>>>(pkeys, ptrie, np, w, tp, first);
    RC(st_scan_u32(ctx, first, bpos, np + 1));
    uint32_t E = 0;
    CU(cudaMemcpyAsync(&E, bpos + np, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    ctx->stats.launches += 2;
    ctx->stats.d2h_bytes += 4;
    uint32_t *etrie, *elo, *ecnt, *estart, *seg_off;
    uint8_t* roots;
    RC(carve(ctx, st->forest, [&](Carve& c) {
        etrie = c.take<uint32_t>(E + 1); elo = c.take<uint32_t>(E + 1); ecnt = c.take<uint32_t>(E + 2); estart = c.take<uint32_t>(E + 1);
        seg_off = c.take<uint32_t>(E + 2); roots = c.take<uint8_t>(32ull * E + 32);
    }));
    wit_bucket_kernel<<<grid1d(dev, np + 1, 128), 128, 0, s>>>(pkeys, ptrie, np, first, bpos, w, krows, n, S, nS, f.arows, etrie, elo, ecnt, estart);
    RC(st_scan_u32(ctx, ecnt, seg_off, E + 1));
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
        wit_forest_vals_kernel<<<grid1d(dev, mk, 256), 256, 0, s>>>(etrie, seg_of_key, src, voff, mk, krows, (const uint8_t*)sp.arena.ptr, S, fv);
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
        if (mk) RC(ctx->build_forest(fk, fko, fv, voff, mk, seg_off, E, seg_of_key, roots, -1, 0, nullptr, nullptr, estart, &xp));
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
    RC(carve(ctx, st->work, [&](Carve& c) {
        perm = c.take<uint32_t>(ne + 1); keep = c.take<uint32_t>(ne + 2); kidx = c.take<uint32_t>(ne + 2);
        size = c.take<uint64_t>(ne + 2); offs = c.take<uint64_t>(ne + 2);
    }));
    RC(ctx->sort_by_segment_and_hash(xp.out.digests, nullptr, ne, perm, st->sort));
    wit_unique_kernel<<<grid1d(dev, ne + 1, 256), 256, 0, s>>>(xp.out.digests, xp.out.nodes, perm, ne, keep, size);
    RC(st_scan_u32(ctx, keep, kidx, ne + 1));
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
    CU(cudaStreamSynchronize(s));
    st->wit_n = nn;
    st->wit_bytes = nb;
    st->wit_held = true;
    return PHANT_GPU_OK;
}

} // namespace

namespace {
int rs_refuse_failed(phant_gpu_resident_state* st)
{
    snprintf(st->ctx->last_error, sizeof st->ctx->last_error, "resident state unusable: an earlier apply failed after it began to write");
    return PHANT_GPU_E_CUDA;
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
    st->acct.ctx = ctx; st->acct.kind = 1; st->acct.depth = 0; st->acct.sp = &st->acct_sp;
    st->acct_sp.compact = true;
    st->acct_sp.compact_row = 112; // an account leaf is at most 110 bytes
    memcpy(st->acct_sp.root, EMPTY_ROOT_H, 32);
    *out = st;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_apply(phant_gpu_resident_state* st, const phant_gpu_state_diff* diff, uint8_t out_root[32],
                                              uint8_t* storage_roots32)
{
    if (!st || !diff || !out_root) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    if (st->failed) return rs_refuse_failed(st);
    CU(cudaSetDevice(ctx->device));
    st->drop_witness();
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
    if (!st || depth > 1024) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    if (st->failed) return rs_refuse_failed(st);
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    st->drop_witness();
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
    if (!st || !out_root) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    if (st->failed) return rs_refuse_failed(st);
    if (n_applies > st->journal.size()) return PHANT_GPU_E_INVALID;
    CU(cudaSetDevice(ctx->device));
    st->drop_witness();
    for (uint32_t k = 0; k < n_applies; ++k) { // newest first: each record is replayed by the apply core, from the device
        phant_gpu_resident_state::Record& r = st->journal.back();
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
        st->spare.push_back(r.buf);
        st->journal.pop_back();
    }
    memcpy(out_root, st->acct_sp.root, 32);
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_witness(phant_gpu_resident_state* st, const phant_gpu_state_diff* diff, phant_gpu_witness_size* out)
{
    if (!st || !diff || !out) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    if (st->failed) return rs_refuse_failed(st);
    CU(cudaSetDevice(ctx->device));
    st->drop_witness();
    memset(out, 0, sizeof *out);
    RC(rs_witness(st, diff));
    out->n_nodes = st->wit_n;
    out->nodes_bytes = st->wit_bytes;
    return PHANT_GPU_OK;
}

extern "C" int phant_gpu_resident_state_witness_copy(phant_gpu_resident_state* st, uint8_t* nodes, uint64_t* node_off)
{
    if (!st || !node_off || !st->wit_held) return PHANT_GPU_E_INVALID;
    phant_gpu_ctx* ctx = st->ctx;
    if (st->wit_bytes && !nodes) return PHANT_GPU_E_INVALID;
    if (is_device_ptr(nodes) || is_device_ptr(node_off)) return PHANT_GPU_E_INVALID; // host pointers, as the diff
    CU(cudaSetDevice(ctx->device));
    if (st->wit_n) {
        const uint64_t* d_off = (const uint64_t*)st->wit_res.ptr;
        CU(cudaMemcpyAsync(node_off, d_off, 8ull * (st->wit_n + 1), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaMemcpyAsync(nodes, d_off + st->wit_n + 1, st->wit_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        ctx->stats.d2h_bytes += 8ull * (st->wit_n + 1) + st->wit_bytes;
    } else node_off[0] = 0;
    st->drop_witness();
    return PHANT_GPU_OK;
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
namespace rs_body {
#include "transition.cuh"
}
namespace tn = rs_body::phant;
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

} // namespace

extern "C" int phant_gpu_transition_roots(phant_gpu_ctx* ctx, const phant_gpu_transition* in, const phant_gpu_state_diff* diff,
                                          uint8_t* post_roots32, uint8_t* status, uint8_t* storage_roots32)
{
    if (!ctx || !in || !diff || !post_roots32 || !status) return PHANT_GPU_E_INVALID;
    // ---- host-side checks: nothing is launched, nothing written, on a bad argument ----
    RC(check_diff_host(ctx, diff));
    const uint64_t nb64 = in->n_blocks, nn = in->n_nodes;
    if (nb64 == 0 || nb64 >= (1ull << 28) || !in->pre_roots32 || nn > (1ull << 30) || (nn && !in->node_off)) return PHANT_GPU_E_INVALID;
    for (const void* q : {(const void*)in->nodes, (const void*)in->node_off, (const void*)in->pre_roots32, (const void*)in->account_block,
                          (const void*)post_roots32, (const void*)status, (const void*)storage_roots32})
        if (is_device_ptr(q)) return PHANT_GPU_E_INVALID;
    const uint32_t nb = (uint32_t)nb64, na = (uint32_t)diff->n_accounts, ms = (uint32_t)diff->n_slots;
    uint64_t nodes_total = 0;
    if (nn) {
        for (uint64_t i = 0; i < nn; ++i) if (in->node_off[i + 1] < in->node_off[i]) return PHANT_GPU_E_INVALID;
        nodes_total = in->node_off[nn];
    }
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
    RC(ctx->d_msgs.reserve(ctx, nodes_total + 64));
    RC(ctx->d_off.reserve(ctx, 8 * (nn + 1)));
    static const uint64_t zero2[2] = {0, 0};
    if (nodes_total) CU(cudaMemcpyAsync(ctx->d_msgs.ptr, in->nodes, nodes_total, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ctx->d_off.ptr, nn ? in->node_off : zero2, 8 * (nn + 1), cudaMemcpyHostToDevice, s));
    ctx->stats.h2d_bytes += nodes_total + 8 * (nn + 1) + 40ull * na + 4ull * na + 4ull * n_st + 32ull * nb;
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
        RC(ctx->sort_by_segment_and_hash(dkeys, dseg, nd, dperm, ctx->tr_sort));
        tr_sorted_keys_kernel<<<grid1d(dev, nd, 256), 256, 0, s>>>(dkeys, dseg, dperm, nd, skeys, sseg, counters + 15);
        ctx->stats.launches++;
        uint32_t dup = 0;
        RC(read_u32(ctx, counters + 15, &dup));
        if (dup) return PHANT_GPU_E_INVALID;
    }
    tr_seg_off_kernel<<<grid1d(dev, n_seg + 1, 256), 256, 0, s>>>(sseg, nd, n_seg, key_lo);
    ctx->stats.launches++;

    // ---- the node set, hashed once into W's digest table; the account walk from each block's root (P) ----
    uint32_t capacity = 64;
    while ((uint64_t)capacity < 2 * nn) capacity <<= 1;
    RC(ctx->d_digests.reserve(ctx, 32 * nn + 32));
    RC(ctx->d_summary.reserve(ctx, 4 * nn + 32));
    RC(ctx->d_index.reserve(ctx, 4ull * capacity));
    RC(ctx->hash_csr(d_nodes, d_noff, nn, nodes_total, (uint8_t*)ctx->d_digests.ptr, (uint32_t*)ctx->d_summary.ptr));
    CU(launch_bag_build(s, dev, (const uint8_t*)ctx->d_digests.ptr, nn, (uint32_t*)ctx->d_index.ptr, capacity));
    if (nn) ctx->stats.launches++;
    const uint8_t* digests = (const uint8_t*)ctx->d_digests.ptr;
    const tn::Bag bag{(const uint32_t*)ctx->d_index.ptr, capacity - 1};
    uint8_t* acc_roots = rec;
    uint8_t* acc_status = rec + 32ull * na;
    if (na) {
        CU(launch_read_accounts(s, dev, na, d_nodes, d_noff, digests, (const uint32_t*)ctx->d_summary.ptr, (const uint32_t*)ctx->d_index.ptr, capacity,
                                dd.akeys, d_aroots, na, nullptr, nullptr, 0, acc_roots, acc_status, StateOut{}));
        tr_block_init_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(acc_status, d_ablock, na, bflags);
        ctx->stats.launches += 2;
    }

    // ---- expand the paths of the listed keys, one level per launch ----
    RC(ctx->tr_front[0].reserve(ctx, sizeof(TFront) * (n_seg + 1)));
    tr_front_init_kernel<<<grid1d(dev, n_seg, 256), 256, 0, s>>>(g, n_seg, bflags, d_pre, dd.aflags, acc_status, acc_roots, key_lo,
                                                                 (TFront*)ctx->tr_front[0].ptr, counters);
    ctx->stats.launches++;
    uint32_t h[2] = {0, 0};
    RC(read_u32(ctx, counters, h, 2));
    uint32_t cur_n = h[0], n_items = 0, levels = 0;
    int cur = 0;
    while (cur_n) {
        if (++levels > 70) return PHANT_GPU_E_CUDA; // cannot happen: every level consumes at least one of the 64 nibbles
        RC(ctx->tr_front[1 - cur].reserve(ctx, sizeof(TFront) * 16ull * cur_n));
        RC(grow_keep(ctx, ctx->tr_items, sizeof(TItem) * (uint64_t)n_items, sizeof(TItem) * ((uint64_t)n_items + cur_n + nd + 1)));
        CU(cudaMemsetAsync(counters, 0, 4, s));
        tr_expand_kernel<<<grid1d(dev, cur_n, 128), 128, 0, s>>>(d_nodes, d_noff, digests, bag, skeys, (const TFront*)ctx->tr_front[cur].ptr, cur_n,
                                                                 (TFront*)ctx->tr_front[1 - cur].ptr, (TItem*)ctx->tr_items.ptr, counters, g, bflags);
        ctx->stats.launches++;
        RC(read_u32(ctx, counters, h, 2));
        cur_n = h[0];
        n_items = h[1];
        cur = 1 - cur;
    }

    // ---- the diff's items beside the witness's; sort; replace, delete, drop failed blocks ----
    RC(grow_keep(ctx, ctx->tr_items, sizeof(TItem) * (uint64_t)n_items, sizeof(TItem) * ((uint64_t)n_items + nd + 1)));
    TItem* items = (TItem*)ctx->tr_items.ptr;
    if (nd) {
        tr_diff_items_kernel<<<grid1d(dev, nd, 256), 256, 0, s>>>(dd, d_ablock, d_segacc, n_st, items + n_items);
        ctx->stats.launches++;
    }
    const uint32_t n = n_items + nd;
    uint8_t *ikeys, *ckeys, *cache, *st_roots, *acc_out;
    uint32_t *iseg, *iperm, *keep, *pos, *cidx, *cseg, *mv_item, *mv_pl, *key_off, *seg_off, *acc_seg_off;
    uint64_t *mv_size, *mv_off, *voff;
    RC(carve(ctx, ctx->tr_work, [&](Carve& c) {
        ikeys = c.take<uint8_t>(32ull * n); iseg = c.take<uint32_t>(n); iperm = c.take<uint32_t>(n);
        keep = c.take<uint32_t>(n + 1); pos = c.take<uint32_t>(n + 1);
        cidx = c.take<uint32_t>(n); ckeys = c.take<uint8_t>(32ull * n); cseg = c.take<uint32_t>(n); cache = c.take<uint8_t>(33ull * n);
        mv_item = c.take<uint32_t>(n); mv_pl = c.take<uint32_t>(n); mv_size = c.take<uint64_t>(n + 1); mv_off = c.take<uint64_t>(n + 1);
        voff = c.take<uint64_t>(n + 1); key_off = c.take<uint32_t>(n + 1);
        seg_off = c.take<uint32_t>(n_seg + 1); acc_seg_off = c.take<uint32_t>(nb + 1);
        st_roots = c.take<uint8_t>(32ull * (n_st + 1)); acc_out = c.take<uint8_t>(32ull * nb);
    }));
    uint32_t m = 0;
    if (n) {
        tr_item_keys_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(items, n, ikeys, iseg);
        ctx->stats.launches++;
        RC(ctx->sort_by_segment_and_hash(ikeys, iseg, n, iperm, ctx->tr_sort));
        tr_classify_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(items, iperm, n, g, bflags, keep);
        CU(cudaMemsetAsync(keep + n, 0, 4, s));
        RC(st_scan_u32(ctx, keep, pos, n + 1));
        tr_compact_kernel<<<grid1d(dev, n, 256), 256, 0, s>>>(items, iperm, keep, pos, n, cidx, ckeys, cseg);
        ctx->stats.launches += 3;
        RC(read_u32(ctx, pos + n, &m));
    }

    // ---- where each stub hangs; the nodes of the stubs the rebuild moves up, encoded and hashed ----
    if (m) {
        tr_place_kernel<<<grid1d(dev, m, 128), 128, 0, s>>>(items, cidx, ckeys, cseg, m, d_nodes, d_noff, digests, bag, g, bflags, cache, mv_item, mv_pl,
                                                            mv_size, counters + 2);
        ctx->stats.launches++;
        uint32_t mv = 0;
        RC(read_u32(ctx, counters + 2, &mv));
        if (mv) {
            RC(scan_sizes(ctx, mv_size, mv_off, mv));
            uint64_t total = 0;
            CU(cudaMemcpyAsync(&total, mv_off + mv, 8, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            uint8_t *arena, *dg;
            RC(carve(ctx, ctx->tr_vals, [&](Carve& c) { arena = c.take<uint8_t>(total + 64); dg = c.take<uint8_t>(32ull * mv); }));
            tr_collapse_encode_kernel<<<grid1d(dev, mv, 128), 128, 0, s>>>(items, cidx, mv_item, mv_pl, mv, mv_off, arena, d_nodes, d_noff, digests, bag);
            RC(ctx->hash_csr(arena, mv_off, mv, total, dg));
            tr_collapse_cache_kernel<<<grid1d(dev, mv, 256), 256, 0, s>>>(items, cidx, mv_item, mv_pl, mv_off, mv, dg, g, bflags, cache);
            ctx->stats.launches += 3;
        }
    }

    // ---- leaf values; the storage forest; account bodies with the new storage roots; the account forest ----
    if (na) {
        iota_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(acc_iota, na);
        account_size_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(dd.nonce, dd.bal, acc_iota, na, asize);
        ctx->stats.launches += 2;
        RC(scan_sizes(ctx, asize, body_off, na));
    }
    uint64_t vtotal = 0;
    if (m) {
        tr_val_size_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(items, cidx, m, dd.svals, asize, mv_size);
        ctx->stats.launches++;
        RC(scan_sizes(ctx, mv_size, voff, m));
        CU(cudaMemcpyAsync(&vtotal, voff + m, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    uint64_t btotal = 0;
    if (na) {
        CU(cudaMemcpyAsync(&btotal, body_off + na, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    uint8_t *arena, *bodies;
    RC(carve(ctx, ctx->tr_vals, [&](Carve& c) { arena = c.take<uint8_t>(vtotal); bodies = c.take<uint8_t>(btotal); }));
    tr_val_fill_kernel<<<grid1d(dev, m + 1, 256), 256, 0, s>>>(items, cidx, m, d_nodes, dd.svals, voff, arena, key_off);
    tr_seg_off_kernel<<<grid1d(dev, n_seg + 1, 256), 256, 0, s>>>(cseg, m, n_seg, seg_off);
    ctx->stats.launches += 2;
    uint32_t m_st = 0;
    RC(read_u32(ctx, seg_off + n_st, &m_st));
    if (n_st) RC(ctx->build_forest(ckeys, key_off, arena, voff, m_st, seg_off, n_st, cseg, st_roots, -1, 0, cache, nullptr));
    if (na) {
        tr_sroot_kernel<<<grid1d(dev, na, 256), 256, 0, s>>>(dd.aflags, na, d_segacc, st_roots, sroot);
        account_fill_kernel<<<grid1d(dev, na + 1, 256), 256, 0, s>>>(dd.nonce, dd.bal, sroot, dd.code, dd.akeys, acc_iota, na, body_off, akeys_scratch,
                                                                   akoff_scratch, bodies);
        ctx->stats.launches += 2;
        if (m) {
            tr_acc_vals_kernel<<<grid1d(dev, m, 256), 256, 0, s>>>(items, cidx, m, body_off, bodies, voff, arena);
            ctx->stats.launches++;
        }
    }
    tr_rebase_kernel<<<grid1d(dev, nb + 1, 256), 256, 0, s>>>(seg_off + n_st, nb + 1, m_st, acc_seg_off);
    ctx->stats.launches++;
    RC(ctx->build_forest(ckeys, key_off + m_st, arena, voff + m_st, m - m_st, acc_seg_off, nb, cseg + m_st, acc_out, -1, 0, cache + 33ull * m_st, nullptr));

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
