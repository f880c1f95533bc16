/* ctrie.c -- TEST INFRASTRUCTURE (see oracle.h).  Resident complete 16-ary trie + dirty-frontier update
 * (BASELINE.json config "state-root recompute: 100k dirty leaves into 16M-node trie").
 *
 * phant has no resident trie (src/state/statedb.zig:16-30 is a hash map and the root check is disabled,
 * src/blockchain/blockchain.zig:83-85); this is the CPU statement of the frontier recompute the
 * north star asks for.  Shape: `depth` branch levels, 16^depth leaves, every branch full, so every
 * branch node is the 532-byte encoding of src/mpt/mpt.zig:218-247 with 16 hashed children and an empty
 * value, and a leaf is rlp([hp(key nibbles [depth,64), leaf), value]) (mpt.zig:255-281).
 * Untouched leaf hashes come from the PRNG (stream tag 0xC4, index = leaf position).
 */
#include "oracle.h"
#include "rlp.h"
#include <stdlib.h>

struct oracle_ctrie {
    uint32_t depth;
    uint8_t** level; /* level[l] = 16^l hashes, l = 0..depth */
};

static inline uint64_t sm64(uint64_t* s)
{
    uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static inline uint64_t stream_init(uint64_t seed, uint64_t tag, uint64_t index)
{
    uint64_t s = seed ^ (tag * 0xA24BAED4963EE407ull) ^ (index * 0xD1342543DE82EF95ull);
    (void)sm64(&s);
    return s;
}

static void hash_branch(const uint8_t* children /* 16 x 32 */, uint8_t out[32])
{
    uint8_t node[532];
    node[0] = 0xf9; node[1] = 0x02; node[2] = 0x11;
    for (int s = 0; s < 16; ++s) {
        node[3 + 33 * s] = 0xa0;
        memcpy(node + 4 + 33 * s, children + 32 * s, 32);
    }
    node[531] = 0x80;
    oracle_keccak256(node, 532, out);
}

oracle_ctrie* oracle_ctrie_open(uint32_t depth, uint64_t seed)
{
    oracle_ctrie* t = calloc(1, sizeof *t);
    t->depth = depth;
    t->level = calloc(depth + 1, sizeof *t->level);
    uint64_t cnt = 1;
    for (uint32_t l = 0; l <= depth; ++l) { t->level[l] = malloc(32 * cnt); cnt *= 16; }
    uint64_t n_leaves = cnt / 16;
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < (int64_t)n_leaves; ++j) {
        uint64_t s = stream_init(seed, 0xC4, (uint64_t)j);
        for (int w = 0; w < 4; ++w) {
            uint64_t v = sm64(&s);
            for (int b = 0; b < 8; ++b) t->level[depth][32 * j + 8 * w + b] = (uint8_t)(v >> (8 * b));
        }
    }
    for (int l = (int)depth - 1; l >= 0; --l) {
        uint64_t n = 1;
        for (int k = 0; k < l; ++k) n *= 16;
#pragma omp parallel for schedule(static)
        for (int64_t j = 0; j < (int64_t)n; ++j) hash_branch(t->level[l + 1] + 512 * j, t->level[l] + 32 * j);
    }
    return t;
}

void oracle_ctrie_root(const oracle_ctrie* t, uint8_t out_root[32]) { memcpy(out_root, t->level[0], 32); }

static int cmp_u64(const void* a, const void* b)
{
    uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? -1 : x > y;
}

void oracle_ctrie_update(oracle_ctrie* t, const uint8_t* keys32, const uint8_t* leaf_vals, const uint32_t* val_off,
                         uint64_t n_dirty, uint8_t out_root[32])
{
    uint32_t L = t->depth;
    uint64_t* idx = malloc((n_dirty + 1) * sizeof *idx);
    /* one leaf buffer for the whole call, sized for the longest value: list header (<= 9) + hp string (<= 34) + value
     * header (<= 9) + value */
    uint64_t max_vl = 0;
    for (uint64_t k = 0; k < n_dirty; ++k)
        if (val_off[k + 1] - val_off[k] > max_vl) max_vl = val_off[k + 1] - val_off[k];
    uint8_t* node = malloc(max_vl + 64);
    for (uint64_t k = 0; k < n_dirty; ++k) {
        const uint8_t* key = keys32 + 32 * k;
        uint64_t pos = 0;
        for (uint32_t i = 0; i < L; ++i) pos = pos * 16 + ((i & 1) ? (key[i >> 1] & 15) : (key[i >> 1] >> 4));
        idx[k] = pos;
        /* leaf = rlp([hp(nibbles[L..64), leaf), value]) */
        uint8_t hp[33];
        uint32_t cnt = 64 - L, o = 0, i = L;
#define KN(q) (((q) & 1) ? (key[(q) >> 1] & 15) : (key[(q) >> 1] >> 4))
        if (cnt & 1) { hp[o++] = (uint8_t)(0x30 | KN(i)); i++; } else hp[o++] = 0x20;
        for (; i < 64; i += 2) hp[o++] = (uint8_t)((KN(i) << 4) | KN(i + 1));
        const uint8_t* v = leaf_vals + val_off[k];
        uint64_t vl = val_off[k + 1] - val_off[k];
        uint64_t payload = rlp_str_size(hp, o) + rlp_str_size(v, vl);
        uint64_t w = rlp_put_list_hdr(node, payload);
        w += rlp_put_str(node + w, hp, o);
        w += rlp_put_str(node + w, v, vl);
        oracle_keccak256(node, w, t->level[L] + 32 * pos);
    }
    free(node);
    uint64_t n = n_dirty;
    for (int l = (int)L - 1; l >= 0; --l) {
        for (uint64_t k = 0; k < n; ++k) idx[k] >>= 4;
        qsort(idx, n, sizeof *idx, cmp_u64);
        uint64_t u = 0;
        for (uint64_t k = 0; k < n; ++k) if (k == 0 || idx[k] != idx[k - 1]) idx[u++] = idx[k];
        n = u;
        for (uint64_t k = 0; k < n; ++k) hash_branch(t->level[l + 1] + 512 * idx[k], t->level[l] + 32 * idx[k]);
    }
    free(idx);
    memcpy(out_root, t->level[0], 32);
}

void oracle_ctrie_free(oracle_ctrie* t)
{
    if (!t) return;
    for (uint32_t l = 0; l <= t->depth; ++l) free(t->level[l]);
    free(t->level);
    free(t);
}
